"""The native UNet step with FreeU off and on.

    python tests/freeu_bench.py [--iters N] [--warmup W] [--rounds R]

Seeded weights (oracle/unet_oracle.py), B = 2 (one image with classifier-free guidance): SD-1.5 at 64^2 latents in
fp16 with (s1, s2, b1, b2) = (0.9, 0.2, 1.2, 1.4), SDXL at 128^2 in bf16 with (0.6, 0.4, 1.1, 1.2).  One compiled
UNet per model; each round times N back-to-back calls with FreeU off, then N with it on (diffusers'
``enable_freeu`` / ``disable_freeu`` between them), with CUDA events after W warm-up calls, so both settings share
the card's state.  Reports the median over R rounds and the spread (max - min) of each.  Prints one JSON line with
the GPU's name and power limit, read in the same process."""
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

from oracle import freeu_oracle as fo  # noqa: E402
from oracle import unet_oracle as uo  # noqa: E402
from t2i_adapter_bench import _unet_kw  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

CASES = (("SD-1.5", uo.sd15_config, 64, torch.float16, (0.9, 0.2, 1.2, 1.4)),
         ("SDXL", uo.sdxl_config, 128, torch.bfloat16, (0.6, 0.4, 1.1, 1.2)))


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args(argv)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    res = dict(_gpu_info(), what="UNet step (B=2), FreeU off vs on, alternated rounds", iters=args.iters,
               warmup=args.warmup, rounds=args.rounds, cases=[])
    for name, cfg_f, lat, dt, vals in CASES:
        cfg, b = cfg_f(), 2
        m = uo.build_unet(cfg, seed=1, dtype=dt, device="cuda")
        unet = compile_unet(m, cc)
        g = torch.Generator(device="cuda").manual_seed(0)
        sample = torch.randn(b, 4, lat, lat, device="cuda", generator=g).to(dt)
        ehs = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
        t = torch.tensor(500, device="cuda")
        kw = _unet_kw(cfg, b, lat, dt, g)
        off, on = [], []
        for _ in range(args.rounds):
            fo.disable_freeu(m)
            off.append(_time(lambda: unet(sample, t, ehs, **kw), args.iters, args.warmup))
            fo.enable_freeu(m, *vals)
            on.append(_time(lambda: unet(sample, t, ehs, **kw), args.iters, args.warmup))
        m_off, m_on = statistics.median(off), statistics.median(on)
        res["cases"].append({"model": name, "dtype": str(dt).replace("torch.", ""), "batch": b, "latent": lat,
                             "freeu": vals, "off_step_ms": m_off, "on_step_ms": m_on,
                             "off_spread_ms": max(off) - min(off), "on_spread_ms": max(on) - min(on),
                             "overhead_pct": 100 * (m_on - m_off) / m_off, "plans": len(unet.forward._cached)})
        del unet, m
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
