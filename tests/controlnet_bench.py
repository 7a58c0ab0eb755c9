"""Native ControlNet (+ UNet) step vs the same pair run eagerly in fp16 (PyTorch library kernels) under a CUDA graph.

    python tests/controlnet_bench.py [--iters N] [--warmup W]

Seeded weights (oracle/controlnet_oracle.py, oracle/unet_oracle.py, no zero-initialised layers), B = 2:
SD-1.5 at 512^2 in fp16 and SDXL at 1024^2 in bf16 on the native side.  Timed with CUDA events over N
back-to-back calls after W warm-up calls:
  * native_controlnet_ms: `compile_controlnet(m)(...)` (input copies, graph replay, output clones);
  * native_step_ms: that call followed by the compiled UNet taking its residuals;
  * eager_graph_step_ms: the same ControlNet + UNet pair in fp16, eager modules captured as one CUDA graph;
  * embedding_share: the conditioning embedding's launches of the native plan (timed alone, replayed
    back to back) over native_controlnet_ms;
  * max_abs_diff_vs_eager: native step output vs the eager pair's, same inputs.
Prints one JSON line with the GPU's name and power limit, read in the same process."""
import argparse
import json
import os
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HERE = os.path.dirname(os.path.abspath(__file__))
for p in (_ROOT, _HERE, os.path.join(_ROOT, "stable-fast_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import controlnet_oracle as co  # noqa: E402
from oracle import unet_oracle as uo  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

CASES = (("SD-1.5", co.sd15_config, uo.sd15_config, 64, torch.float16),
         ("SDXL", co.sdxl_config, uo.sdxl_config, 128, torch.bfloat16))


def _inputs(cfg, b, lat, dt):
    g = torch.Generator(device="cuda").manual_seed(0)
    sample = torch.randn(b, 4, lat, lat, device="cuda", generator=g).to(dt)
    cond = torch.rand(b, 3, 8 * lat, 8 * lat, device="cuda", generator=g).to(dt)
    ehs = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        kw["added_cond_kwargs"] = dict(text_embeds=torch.randn(b, 1280, device="cuda", generator=g).to(dt),
                                       time_ids=torch.tensor([[8 * lat, 8 * lat, 0, 0, 8 * lat, 8 * lat]] * b,
                                                             device="cuda", dtype=torch.float32))
    return sample, torch.tensor(500, device="cuda"), ehs, cond, kw


def _cast_kw(kw, dt):
    return {k: {kk: (vv.to(dt) if vv.dtype != torch.float32 else vv) for kk, vv in v.items()} for k, v in kw.items()}


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_controlnet, compile_unet
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args(argv)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    res = dict(_gpu_info(), what="ControlNet + UNet step, B=2, native vs eager fp16 under a CUDA graph",
               iters=args.iters, warmup=args.warmup, cases=[])
    b = 2
    for name, cn_cfg_f, unet_cfg_f, lat, dt in CASES:
        cn_cfg, unet_cfg = cn_cfg_f(), unet_cfg_f()
        cn = compile_controlnet(co.build_controlnet(cn_cfg, seed=0, dtype=dt, device="cuda"), cc)
        unet = compile_unet(uo.build_unet(unet_cfg, seed=1, dtype=dt, device="cuda"), cc)
        sample, t, ehs, cond, kw = _inputs(cn_cfg, b, lat, dt)

        def native_cn():
            return cn(sample, t, ehs, cond, conditioning_scale=0.8, return_dict=False, **kw)

        def native_step():
            down, mid = native_cn()
            return unet(sample, t, ehs, down_block_additional_residuals=down, mid_block_additional_residual=mid,
                        **kw).sample

        ms_cn = _time(native_cn, args.iters, args.warmup)
        ms_step = _time(native_step, args.iters, args.warmup)
        with torch.no_grad():
            native_out = native_step().float()
        # the conditioning embedding's launches alone, on the plan the native call just ran
        plan = next(iter(cn.forward._cached.values())).plan
        emb_ops = [op for op in plan.ops if op.name.startswith("controlnet_cond_embedding")]
        stream = torch.cuda.current_stream().cuda_stream

        def emb():
            for op in emb_ops:
                op.launch(stream)
        ms_emb = _time(emb, args.iters, args.warmup)
        del plan, emb_ops
        del cn, unet
        torch.cuda.empty_cache()

        # eager pair in fp16 under one CUDA graph
        h16 = torch.float16
        ecn = co.build_controlnet(cn_cfg, seed=0, dtype=h16, device="cuda")
        eunet = uo.build_unet(unet_cfg, seed=1, dtype=h16, device="cuda")
        es, ee, ec, ekw = sample.to(h16), ehs.to(h16), cond.to(h16), _cast_kw(kw, h16)

        def eager_step():
            down, mid = ecn(es, t, ee, ec, conditioning_scale=0.8, return_dict=False, **ekw)
            return eunet(es, t, ee, down_block_additional_residuals=down, mid_block_additional_residual=mid,
                         **ekw).sample

        with torch.no_grad():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    eager_step()
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                eager_out = eager_step()
            ms_eager = _time(g.replay, args.iters, args.warmup)
            g.replay()
            torch.cuda.synchronize()
            diff = (native_out - eager_out.float()).abs().max().item()
            ref_max = eager_out.float().abs().max().item()
        res["cases"].append({"model": name, "dtype": str(dt).replace("torch.", ""), "batch": b,
                             "image": 8 * lat, "latent": lat, "native_controlnet_ms": ms_cn,
                             "native_step_ms": ms_step, "eager_graph_step_ms": ms_eager,
                             "step_speedup": ms_eager / ms_step, "embedding_ms": ms_emb,
                             "embedding_share": ms_emb / ms_cn, "max_abs_diff_vs_eager": diff,
                             "eager_out_max_abs": ref_max})
        del g, ecn, eunet, eager_out
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
