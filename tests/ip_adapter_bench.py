"""Native UNet step with and without an IP-Adapter vs the oracle UNet with the adapter run eagerly under a CUDA graph.

    python tests/ip_adapter_bench.py [--iters N] [--warmup W]

Seeded weights (oracle/unet_oracle.py + oracle/ip_adapter_oracle.py, one image, 4 image tokens), B = 2:
SD-1.5 at 512^2 in fp16 (ip-adapter_sd15 shape, D_img 1024) and SDXL at 1024^2 in bf16 (ViT-H adapter shape).
Timed with CUDA events over N back-to-back calls after W warm-up calls:
  * native_ms: `compile_unet(m)(...)` of the UNet without the adapter (input copies, graph replay, output clone);
  * native_ip_ms: the same UNet with the adapter loaded and image_embeds passed;
  * eager_graph_ip_ms: the oracle UNet with the adapter, eager modules in the same dtype captured as one CUDA graph;
  * max_abs_diff_vs_eager: native output with the adapter vs the eager graph's, same inputs.
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
from oracle import unet_oracle as uo  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

CASES = (("SD-1.5", uo.sd15_config, 64, torch.float16, 1024),
         ("SDXL", uo.sdxl_config, 128, torch.bfloat16, 1024))


def _inputs(cfg, b, lat, dt, d_img):
    g = torch.Generator(device="cuda").manual_seed(0)
    sample = torch.randn(b, 4, lat, lat, device="cuda", generator=g).to(dt)
    ehs = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        kw = dict(text_embeds=torch.randn(b, 1280, device="cuda", generator=g).to(dt),
                  time_ids=torch.tensor([[8 * lat, 8 * lat, 0, 0, 8 * lat, 8 * lat]] * b, device="cuda",
                                        dtype=torch.float32))
    ip_kw = dict(kw, image_embeds=[torch.randn(b, 1, d_img, device="cuda", generator=g).to(dt)])
    return sample, torch.tensor(500, device="cuda"), ehs, kw, ip_kw


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args(argv)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    res = dict(_gpu_info(), what="UNet step with / without an IP-Adapter, B=2, native vs eager under a CUDA graph",
               iters=args.iters, warmup=args.warmup, cases=[])
    b = 2
    for name, cfg_f, lat, dt, d_img in CASES:
        cfg = cfg_f()
        sample, t, ehs, kw, ip_kw = _inputs(cfg, b, lat, dt, d_img)
        plain = compile_unet(uo.build_unet(cfg, seed=1, dtype=dt, device="cuda"), cc)
        ms_plain = _time(lambda: plain(sample, t, ehs, added_cond_kwargs=kw or None).sample, args.iters, args.warmup)
        del plain
        torch.cuda.empty_cache()
        unet = ipo.load_ip_adapter(uo.build_unet(cfg, seed=1, dtype=dt, device="cuda"), d_img, seed=2, scale=0.6)
        eager = ipo.load_ip_adapter(uo.build_unet(cfg, seed=1, dtype=dt, device="cuda"), d_img, seed=2, scale=0.6)
        fast = compile_unet(unet, cc)

        def native():
            return fast(sample, t, ehs, added_cond_kwargs=ip_kw).sample
        ms_ip = _time(native, args.iters, args.warmup)
        native_out = native().float()
        del fast, unet
        torch.cuda.empty_cache()
        with torch.no_grad():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    eager(sample, t, ehs, added_cond_kwargs=ip_kw)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                eager_out = eager(sample, t, ehs, added_cond_kwargs=ip_kw).sample
            ms_eager = _time(g.replay, args.iters, args.warmup)
            g.replay()
            torch.cuda.synchronize()
            diff = (native_out - eager_out.float()).abs().max().item()
            ref_max = eager_out.float().abs().max().item()
        res["cases"].append({"model": name, "dtype": str(dt).replace("torch.", ""), "batch": b, "image": 8 * lat,
                             "latent": lat, "image_tokens": 4, "native_ms": ms_plain, "native_ip_ms": ms_ip,
                             "ip_overhead_ms": ms_ip - ms_plain, "eager_graph_ip_ms": ms_eager,
                             "speedup_vs_eager": ms_eager / ms_ip, "max_abs_diff_vs_eager": diff,
                             "eager_out_max_abs": ref_max})
        del g, eager, eager_out
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
