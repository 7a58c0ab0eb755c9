"""The native UNet step of the inpainting and LCM UNets against the plain UNet of the same model.

    python tests/lcm_inpaint_bench.py [--iters N] [--warmup W] [--rounds R]

Seeded weights (oracle/unet_oracle.py): SD-1.5 at 64^2 latents in fp16 and SDXL at 128^2 in bf16.  Inpainting at
B = 2 (one image with classifier-free guidance; 9 input channels: conv_in is a wide im2col + a K = 128 GEMM), LCM at
B = 1 (LCM pipelines run without classifier-free guidance; one more batch-row linear, cond_proj, on the time-embedding
branch).  Each round times N back-to-back calls of the plain compiled UNet, then N of the variant, with CUDA events
after W warm-up calls, so both share the card's state.  Reports the median over R rounds and the spread (max - min)
of each.  Prints one JSON line with the GPU's name and power limit, read in the same process."""
import argparse
import json
import os
import statistics
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HERE = os.path.dirname(os.path.abspath(__file__))
for p in (_ROOT, _HERE, os.path.join(_ROOT, "stable-fast_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import lcm_inpaint_oracle as lio  # noqa: E402
from oracle import unet_oracle as uo  # noqa: E402
from t2i_adapter_bench import _unet_kw  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

CASES = (("SD-1.5", "inpaint", uo.sd15_config, lio.sd15_inpaint_config, 64, torch.float16, 2),
         ("SDXL", "inpaint", uo.sdxl_config, lio.sdxl_inpaint_config, 128, torch.bfloat16, 2),
         ("SD-1.5", "lcm", uo.sd15_config, lio.lcm_sd15_config, 64, torch.float16, 1),
         ("SDXL", "lcm", uo.sdxl_config, lio.lcm_sdxl_config, 128, torch.bfloat16, 1))


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args(argv)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    res = dict(_gpu_info(), what="UNet step, plain vs inpainting (B=2) / LCM (B=1), alternated rounds",
               iters=args.iters, warmup=args.warmup, rounds=args.rounds, cases=[])
    for name, kind, plain_f, var_f, lat, dt, b in CASES:
        calls = []
        for cfg in (plain_f(), var_f()):
            unet = compile_unet(lio.build_unet(cfg, seed=1, dtype=dt, device="cuda"), cc)
            g = torch.Generator(device="cuda").manual_seed(0)
            sample = torch.randn(b, cfg.in_channels, lat, lat, device="cuda", generator=g).to(dt)
            ehs = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
            kw = _unet_kw(cfg, b, lat, dt, g)
            if getattr(cfg, "time_cond_proj_dim", None):
                kw["timestep_cond"] = torch.randn(b, cfg.time_cond_proj_dim, device="cuda", generator=g).to(dt)
            t = torch.tensor(500, device="cuda")
            calls.append(lambda unet=unet, sample=sample, ehs=ehs, kw=kw, t=t: unet(sample, t, ehs, **kw))
        plain, var = [], []
        for _ in range(args.rounds):
            plain.append(_time(calls[0], args.iters, args.warmup))
            var.append(_time(calls[1], args.iters, args.warmup))
        m_p, m_v = statistics.median(plain), statistics.median(var)
        res["cases"].append({"model": name, "variant": kind, "dtype": str(dt).replace("torch.", ""), "batch": b,
                             "latent": lat, "plain_step_ms": m_p, "variant_step_ms": m_v,
                             "plain_spread_ms": max(plain) - min(plain), "variant_spread_ms": max(var) - min(var),
                             "overhead_us": 1000 * (m_v - m_p), "overhead_pct": 100 * (m_v - m_p) / m_p})
        del calls
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
