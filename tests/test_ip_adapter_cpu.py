"""Host-side checks of the native IP-Adapter: the oracle adapter's parameters against the spec (totals pinned),
the dry launch schedules with and without image tokens, a float64 restatement of the fused attention against
the oracle processor, the new parameter struct's layout, the C ABI's validation of sfb_attention_ip, and every
refusal by name."""
import ctypes
import math
import os
import subprocess
import types

import pytest
import torch
import torch.nn as nn

from oracle import controlnet_oracle as co
from oracle import ip_adapter_oracle as ipo
from oracle import unet_oracle as uo
from sfast_b200 import _lib
from sfast_b200.plan import PackedWeights, UNetPlan
from sfast_b200.runtime import CompiledUNet
from sfast_b200.unet_spec import (controlnet_spec_from_config, ip_adapter_geometry, ip_adapter_spec, param_shapes,
                                  spec_from_config)
from test_host_logic import _DUMMY_PTR, _validate_plan_on_cpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")
CFGS = {"tiny": uo.tiny_config, "sd15": uo.sd15_config, "sdxl": uo.sdxl_config}


def _ip_count(shapes):
    return sum(math.prod(v) for k, v in shapes.items() if k.startswith("encoder_hid_proj.") or ".processor." in k)


def _meta_unet(cfgf, d_img):
    with torch.device("meta"):
        m = uo.UNet2DConditionModel(cfgf())
    return ipo.load_ip_adapter(m, d_img)


@pytest.mark.parametrize("cfg,d_img,layers,total", [("sd15", 1024, 16, 22_319_616), ("sdxl", 1024, 70, 349_188_096),
                                                    ("sdxl", 1280, 70, 351_285_248)])
def test_parameter_totals_are_pinned_and_the_oracle_matches_the_spec(cfg, d_img, layers, total):
    m = _meta_unet(CFGS[cfg], d_img)
    assert ipo.ip_adapter_param_count(m) == total
    spec = spec_from_config(m.config)
    spec.ip = ip_adapter_spec(m, spec)
    assert len(spec.ip.layers) == layers and (spec.ip.image_embed_dim, spec.ip.tokens) == (d_img, 4)
    shapes = param_shapes(spec)
    assert _ip_count(shapes) == total
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == {k: tuple(v) for k, v in shapes.items()}
    assert "encoder_hid_proj.image_projection_layers.0.image_embeds.weight" in got
    assert "mid_block.attentions.0.transformer_blocks.0.attn2.processor.to_k_ip.0.weight" in got


def _dry(cfg, b, h, w, ip_len, d_img=64, dt=torch.float16, with_ip=True):
    spec = spec_from_config(CFGS[cfg]())
    if with_ip:
        spec.ip = ip_adapter_geometry(spec, d_img)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    return UNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w, ip_len=ip_len)


def _sequence(plan):
    return [(op.name, op.fn.name if op.fn is not None else None) for op in plan.all_ops()]


@pytest.mark.parametrize("cfg,b,h,w,d_img", [("tiny", 2, 32, 32, 64), ("sd15", 2, 64, 64, 1024),
                                             ("sdxl", 1, 128, 128, 1280)])
def test_launch_counts_and_an_unchanged_schedule_without_image_tokens(cfg, b, h, w, d_img):
    base = _dry(cfg, b, h, w, 0, d_img, with_ip=False)
    assert _sequence(_dry(cfg, b, h, w, 0, d_img)) == _sequence(base)
    n_cross = len(spec_from_config(CFGS[cfg]()).cross_attention_layers())
    for ip_len in (4, 16):
        plan = _dry(cfg, b, h, w, ip_len, d_img)
        names = [n for n, _ in _sequence(plan)]
        fns = [f for _, f in _sequence(plan)]
        # projection + LayerNorm + one K/V GEMM per cross-attention, all on the side stream
        assert len(names) == len(base.all_ops()) + 2 + n_cross
        assert sum(n.endswith(".ip_kv") for n in names) == n_cross
        assert fns.count("sfb_attention_ip") == n_cross
        assert fns.count("sfb_attention") == [f for _, f in _sequence(base)].count("sfb_attention") - n_cross
        side = {op.name for op in plan.side_ops}
        assert {"encoder_hid_proj.image_projection_layers.0.image_embeds",
                "encoder_hid_proj.image_projection_layers.0.norm"} <= side
        assert all(n in side for n in names if n.endswith(".ip_kv"))
        assert tuple(plan.image_embeds_in.shape) == (b * ip_len // 4, d_img)
        assert tuple(plan.ip_scale_in.shape) == (n_cross,)
        ops_ = [op for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_attention_ip"]
        assert not any(op.keep[0].ip_scale for op in ops_)  # dry: slices of one meta buffer (address 0)
        assert all(op.keep[0].seq_ip == ip_len and op.keep[0].k_ip_rows == ip_len for op in ops_)


@_NO_GPU
def test_dry_ip_plans_pass_host_validation():
    lib = _lib.lib()
    for cfg, b, h, w, d_img, ip_len in (("tiny", 2, 32, 32, 64, 4), ("sd15", 2, 64, 64, 1024, 16),
                                        ("sdxl", 2, 64, 64, 1024, 4)):
        plan = _dry(cfg, b, h, w, ip_len, d_img)
        n = _validate_plan_on_cpu(plan)
        assert n["sfb_gemm"] > 0
        n_ip = 0
        for op in plan.all_ops():
            if op.fn is not None and op.fn.name == "sfb_attention_ip":
                p = _lib.AttnIpParams()
                ctypes.memmove(ctypes.byref(p), ctypes.byref(op.keep[0]), ctypes.sizeof(p))
                for f in ("tmap_q", "tmap_k", "tmap_vt", "out"):
                    setattr(p.base, f, getattr(p.base, f) or _DUMMY_PTR)
                for f in ("tmap_k_ip", "tmap_vt_ip", "ip_scale"):
                    setattr(p, f, getattr(p, f) or _DUMMY_PTR)
                rc = lib.sfb_attention_ip(ctypes.byref(p), None)
                assert rc == -2, f"{op.name}: {lib.sfb_last_error().decode()}"
                n_ip += 1
        assert n_ip == len(plan.spec.ip.layers)


def test_too_many_image_tokens_are_refused():
    with pytest.raises(NotImplementedError, match="one KV tile"):
        _dry("sd15", 1, 64, 64, 68, 1024)
    with pytest.raises(NotImplementedError, match="one KV tile"):
        _dry("sdxl", 1, 64, 64, 68, 1024)


def fused_attention_reference(q, k, v, k_ip, v_ip, scale):
    """float64 restatement of sfb_attention_ip from include/sfb200.h, element by element: two separate softmaxes
    (row maximum, exponentials, row sum) over the text keys and the image keys."""
    def attn(k_, v_):
        s = q @ k_.transpose(-1, -2) / math.sqrt(q.shape[-1])
        p = torch.exp(s - s.max(-1, keepdim=True).values)
        return (p / p.sum(-1, keepdim=True)) @ v_
    return attn(k, v) + scale * attn(k_ip, v_ip)


@pytest.mark.parametrize("scale", [0.0, 0.6, 1.0, -0.5])
def test_fused_attention_reference_matches_the_oracle_processor(scale):
    torch.manual_seed(1)
    dim, heads, ctx, b, s, n_img = 64, 2, 32, 2, 10, 3
    attn = uo.Attention(dim, heads, ctx).double()
    proc = ipo.IPAdapterAttnProcessor2_0(dim, ctx, (4,), scale).double()
    x, text, ip = torch.randn(b, s, dim).double(), torch.randn(b, 7, ctx).double(), torch.randn(b, n_img, 4, ctx)
    with torch.no_grad():
        got = proc(attn, x, (text, [ip.double()]))

        def split(t):
            return t.view(b, -1, heads, dim // heads).transpose(1, 2)
        ipf = ip.double().reshape(b, n_img * 4, ctx)
        o = fused_attention_reference(split(attn.to_q(x)), split(attn.to_k(text)), split(attn.to_v(text)),
                                      split(proc.to_k_ip[0](ipf)), split(proc.to_v_ip[0](ipf)), scale)
        ref = attn.to_out[0](o.transpose(1, 2).reshape(b, s, dim))
    assert torch.allclose(got, ref, rtol=1e-10, atol=1e-12)


def test_attn_ip_struct_layout_matches_the_header(tmp_path):
    cls, cname = _lib.AttnIpParams, "sfb_attn_ip_params"
    lines = [f'printf("{cname} %zu\\n", sizeof({cname}));']
    for fname, _ in cls._fields_:
        lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sfb200.h"\nint main(void) {\n'
                   + "\n".join(lines) + "\nreturn 0; }\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                       text=True).stdout.strip().splitlines())
    assert int(got[cname]) == ctypes.sizeof(cls)
    for fname, _ in cls._fields_:
        assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, fname
    assert "sfb_attention_ip" in _lib.SYMBOLS


@_NO_GPU
def test_attention_ip_rejects_bad_arguments():
    lib = _lib.lib()

    def call(base=None, **kw):
        p = _lib.AttnIpParams()
        b = p.base
        b.tmap_q = b.tmap_k = b.tmap_vt = b.out = _DUMMY_PTR
        b.batch, b.heads, b.head_dim, b.seq_q, b.seq_kv = 1, 2, 40, 128, 77
        b.q_rows, b.k_rows, b.vt_rows, b.scale, b.kv_tile = 128, 77, 48, 0.15, 128
        p.tmap_k_ip = p.tmap_vt_ip = p.ip_scale = _DUMMY_PTR
        p.seq_ip, p.k_ip_rows = 4, 4
        for k, v in (base or {}).items():
            setattr(b, k, v)
        for k, v in kw.items():
            setattr(p, k, v)
        rc = lib.sfb_attention_ip(ctypes.byref(p), None)
        return rc, lib.sfb_last_error().decode()
    assert call()[0] == -2 and call(seq_ip=128, k_ip_rows=128)[0] == -2 and \
        call(dict(kv_tile=64), seq_ip=64, k_ip_rows=64)[0] == -2
    for kw, what in ((dict(tmap_k_ip=None), "tmap_k_ip"), (dict(ip_scale=None), "ip_scale"),
                     (dict(seq_ip=0), "seq_ip"), (dict(seq_ip=129, k_ip_rows=129), "seq_ip"),
                     (dict(k_ip_rows=3), "k_ip_rows")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, (kw, msg)
    rc, msg = call(dict(kv_tile=64), seq_ip=65, k_ip_rows=65)
    assert rc == -1 and "seq_ip" in msg
    for base, what in ((dict(causal=1, kv_tile=64, seq_q=77), "causal"), (dict(head_dim=48, vt_rows=64), "head_dim"),
                       (dict(vt_rows=64), "vt_rows"), (dict(kv_tile=64, head_dim=80, vt_rows=96), "kv_tile 64")):
        rc, msg = call(base)
        assert rc == -1 and what in msg and "sfb_attention_ip" in msg, (base, msg)


# ---------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------
def _tiny_ip(d_img=64):
    return ipo.load_ip_adapter(uo.build_unet(uo.tiny_config(), seed=0), d_img)


def _renamed(obj, name):
    obj.__class__ = type(name, (type(obj),), {})
    return obj


def test_a_plain_adapter_is_read_from_the_module():
    m = _tiny_ip()
    spec = spec_from_config(m.config)
    ip = ip_adapter_spec(m, spec)
    assert ip == ip_adapter_geometry(spec, 64) and len(ip.layers) == 16


@pytest.mark.parametrize("mutate,match", [
    (lambda m: _renamed(m.encoder_hid_proj.image_projection_layers[0], "IPAdapterPlusImageProjection"),
     "IPAdapterPlusImageProjection"),
    (lambda m: _renamed(m.encoder_hid_proj.image_projection_layers[0], "IPAdapterFaceIDImageProjection"), "FaceID"),
    (lambda m: _renamed(m.encoder_hid_proj.image_projection_layers[0], "IPAdapterFaceIDPlusImageProjection"),
     "FaceID"),
    (lambda m: m.encoder_hid_proj.image_projection_layers.append(m.encoder_hid_proj.image_projection_layers[0]),
     "more than one IP-Adapter"),
    (lambda m: setattr(m, "text_encoder_hid_proj", nn.Linear(4, 4)), "text_encoder_hid_proj"),
    (lambda m: setattr(m.down_blocks[1].attentions[0].transformer_blocks[0].attn2.processor, "scale", [[0.5, 0.7]]),
     "per-image"),
    (lambda m: setattr(m.mid_block.attentions[0].transformer_blocks[0].attn2.processor, "scale", [0.5, 0.5]),
     "one float per layer"),
    (lambda m: m.mid_block.attentions[0].transformer_blocks[0].attn2.processor.to_k_ip.append(nn.Linear(128, 256)),
     "more than one IP-Adapter"),
])
def test_unsupported_adapters_are_refused_by_name(mutate, match):
    m = _tiny_ip()
    mutate(m)
    with pytest.raises(NotImplementedError, match=match):
        ip_adapter_spec(m, spec_from_config(m.config))
    with pytest.raises(NotImplementedError, match=match):
        CompiledUNet(m.config, m.state_dict, module=m)


def test_controlnet_configs_keep_refusing_ip_image_proj():
    cfg = dict(vars(co.sd15_config()), encoder_hid_dim_type="ip_image_proj")
    with pytest.raises(NotImplementedError, match="encoder_hid_dim_type"):
        controlnet_spec_from_config(cfg)
    spec_from_config(dict(vars(uo.sd15_config()), encoder_hid_dim_type="ip_image_proj"))
    with pytest.raises(NotImplementedError, match="encoder_hid_dim_type"):
        spec_from_config(dict(vars(uo.sd15_config()), encoder_hid_dim_type="text_proj"))


def test_call_time_refusals():
    m = _tiny_ip()
    c = CompiledUNet(m.config, m.state_dict, module=m)
    x, t, e = torch.randn(1, 4, 32, 32).half(), torch.tensor(1), torch.randn(1, 77, 128).half()
    emb = [torch.randn(1, 1, 64).half()]
    with pytest.raises(ValueError, match="image_embeds"):
        c(x, t, e)
    with pytest.raises(NotImplementedError, match="ip_adapter_masks"):
        c(x, t, e, added_cond_kwargs=dict(image_embeds=emb), cross_attention_kwargs=dict(ip_adapter_masks=[None]))
    with pytest.raises(NotImplementedError, match="one adapter"):
        c(x, t, e, added_cond_kwargs=dict(image_embeds=emb * 2))
    with pytest.raises(ValueError, match="image_embeds of shape"):
        c(x, t, e, added_cond_kwargs=dict(image_embeds=[torch.randn(1, 1, 32)]))
    m.encoder_hid_proj = ipo.MultiIPAdapterImageProjection([ipo.ImageProjection(64, 128)])
    with pytest.raises(NotImplementedError, match="compile"):
        c(x, t, e, added_cond_kwargs=dict(image_embeds=emb))
    with pytest.raises(NotImplementedError, match="module"):
        CompiledUNet(m.config, m.state_dict)
    # an adapter loaded after compiling a plain UNet
    plain = uo.build_unet(uo.tiny_config(), seed=0)
    c2 = CompiledUNet(plain.config, plain.state_dict, module=plain)
    ipo.load_ip_adapter(plain, 64)
    with pytest.raises(NotImplementedError, match="compile"):
        c2(x, t, e, added_cond_kwargs=dict(image_embeds=emb))


def test_oracle_requires_image_embeds_like_diffusers():
    m = _tiny_ip()
    with pytest.raises(ValueError, match="image_embeds"):
        m(torch.randn(1, 4, 32, 32), torch.tensor(1), torch.randn(1, 77, 128))
    bare = m(torch.randn(1, 4, 32, 32), torch.tensor(1), torch.randn(1, 77, 128),
             added_cond_kwargs=dict(image_embeds=torch.randn(1, 64))).sample
    assert bare.shape == (1, 4, 32, 32) and types.MethodType is type(m.forward)
