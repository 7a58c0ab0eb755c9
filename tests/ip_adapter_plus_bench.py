"""Native UNet step without an adapter, with a plain IP-Adapter and with IP-Adapter Plus, vs the oracle UNet with
the Plus adapter run eagerly under a CUDA graph.

    python tests/ip_adapter_plus_bench.py [--iters N] [--warmup W]

Seeded weights (oracle/unet_oracle.py, oracle/ip_adapter_oracle.py, oracle/ip_adapter_plus_oracle.py), B = 2,
one image: SD-1.5 at 512^2 in fp16 (ip-adapter_sd15 / ip-adapter-plus_sd15 shapes) and SDXL at 1024^2 in bf16
(ip-adapter_sdxl_vit-h / ip-adapter-plus_sdxl_vit-h shapes); Plus takes ViT-H/14 image features [B, 1, 257, 1280].
Timed with CUDA events over N back-to-back calls after W warm-up calls:
  * native_ms: `compile_unet(m)(...)` of the UNet without an adapter (input copies, graph replay, output clone);
  * native_ip_ms: the same with the plain adapter (4 image tokens);
  * native_plus_ms: the same with IP-Adapter Plus (16 image tokens, the Resampler inside the step);
  * eager_graph_plus_ms: the oracle UNet with the Plus adapter, eager modules in the same dtype captured as one
    CUDA graph;
  * max_abs_diff_vs_eager: native Plus output vs the eager graph's, same inputs.
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

from oracle import ip_adapter_oracle as ipo  # noqa: E402
from oracle import ip_adapter_plus_oracle as ipp  # noqa: E402
from oracle import unet_oracle as uo  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

# (name, config, latent size, dtype, plain adapter D_img, Plus D_img, Plus hidden dims)
CASES = (("SD-1.5", uo.sd15_config, 64, torch.float16, 1024, 1280, 768),
         ("SDXL", uo.sdxl_config, 128, torch.bfloat16, 1280, 1280, 1280))
S_IMG = 257


def _inputs(cfg, b, lat, dt, d_plain, d_plus):
    g = torch.Generator(device="cuda").manual_seed(0)
    sample = torch.randn(b, 4, lat, lat, device="cuda", generator=g).to(dt)
    ehs = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        kw = dict(text_embeds=torch.randn(b, 1280, device="cuda", generator=g).to(dt),
                  time_ids=torch.tensor([[8 * lat, 8 * lat, 0, 0, 8 * lat, 8 * lat]] * b, device="cuda",
                                        dtype=torch.float32))
    ip_kw = dict(kw, image_embeds=[torch.randn(b, 1, d_plain, device="cuda", generator=g).to(dt)])
    plus_kw = dict(kw, image_embeds=[torch.randn(b, 1, S_IMG, d_plus, device="cuda", generator=g).to(dt)])
    return sample, torch.tensor(500, device="cuda"), ehs, kw, ip_kw, plus_kw


def _native_ms(unet, cc, args, kw, iters, warmup):
    from sfast.compilers.diffusion_pipeline_compiler import compile_unet
    fast = compile_unet(unet, cc)

    def call():
        return fast(*args, added_cond_kwargs=kw or None).sample
    ms = _time(call, iters, warmup)
    out = call().float()
    return ms, out


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args(argv)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    res = dict(_gpu_info(), what="UNet step without an adapter, with IP-Adapter and with IP-Adapter Plus, B=2, "
               "native vs eager under a CUDA graph", iters=args.iters, warmup=args.warmup, cases=[])
    b = 2
    for name, cfg_f, lat, dt, d_plain, d_plus, dh in CASES:
        cfg = cfg_f()
        sample, t, ehs, kw, ip_kw, plus_kw = _inputs(cfg, b, lat, dt, d_plain, d_plus)
        call = (sample, t, ehs)
        ms_plain, _ = _native_ms(uo.build_unet(cfg, seed=1, dtype=dt, device="cuda"), cc, call, kw, args.iters,
                                 args.warmup)
        torch.cuda.empty_cache()
        unet = ipo.load_ip_adapter(uo.build_unet(cfg, seed=1, dtype=dt, device="cuda"), d_plain, seed=2, scale=0.6)
        ms_ip, _ = _native_ms(unet, cc, call, ip_kw, args.iters, args.warmup)
        del unet
        torch.cuda.empty_cache()
        unet = ipp.load_ip_adapter_plus(uo.build_unet(cfg, seed=1, dtype=dt, device="cuda"), d_plus, dh, seed=3,
                                        scale=0.6)
        ms_plus, native_out = _native_ms(unet, cc, call, plus_kw, args.iters, args.warmup)
        del unet
        torch.cuda.empty_cache()
        eager = ipp.load_ip_adapter_plus(uo.build_unet(cfg, seed=1, dtype=dt, device="cuda"), d_plus, dh, seed=3,
                                         scale=0.6)
        with torch.no_grad():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    eager(sample, t, ehs, added_cond_kwargs=plus_kw)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                eager_out = eager(sample, t, ehs, added_cond_kwargs=plus_kw).sample
            ms_eager = _time(g.replay, args.iters, args.warmup)
            g.replay()
            torch.cuda.synchronize()
            diff = (native_out - eager_out.float()).abs().max().item()
            ref_max = eager_out.float().abs().max().item()
        res["cases"].append({"model": name, "dtype": str(dt).replace("torch.", ""), "batch": b, "image": 8 * lat,
                             "latent": lat, "images": 1, "plain_image_tokens": 4, "plus_image_tokens": 16,
                             "plus_image_features": [S_IMG, d_plus], "plus_hidden_dims": dh,
                             "native_ms": ms_plain, "native_ip_ms": ms_ip, "native_plus_ms": ms_plus,
                             "plus_overhead_ms": ms_plus - ms_plain, "plus_over_plain_ip_ms": ms_plus - ms_ip,
                             "eager_graph_plus_ms": ms_eager, "speedup_vs_eager": ms_eager / ms_plus,
                             "max_abs_diff_vs_eager": diff, "eager_out_max_abs": ref_max})
        del g, eager, eager_out
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
