"""Native VAE encode vs the same AutoencoderKL run eagerly (PyTorch library kernels) under a CUDA graph.

    python tests/vae_encode_bench.py [--iters N] [--warmup W]

SD-1.5 VAE (oracle/vae_encoder_oracle.py, seeded weights), fp16, images in [-1, 1]; both sides are timed with CUDA
events over N back-to-back calls after W warm-up calls: the native side is `compile_vae(m).encode(x)`
(input copy, graph replay, output clone), the eager side is a captured graph of `quant_conv(encoder(x))`.
Prints one JSON line with the GPU's name and power limit, read in the same process."""
import argparse
import json
import os
import subprocess
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (_ROOT, os.path.join(_ROOT, "stable-fast_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import vae_encoder_oracle as veo  # noqa: E402
from oracle import vae_oracle as vo  # noqa: E402

SHAPES = ((1, 512, 512), (4, 512, 512), (1, 576, 1024))


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power, clock = (s.strip() for s in out.strip().split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unread ({exc!r})"}


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_vae
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args(argv)
    dev = "cuda"
    cfg = vo.sd_vae_config()
    eager = veo.build_autoencoder_kl(cfg, seed=0, dtype=torch.float16, device=dev)
    fast = veo.build_autoencoder_kl(cfg, seed=0, dtype=torch.float16, device=dev)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    fast = compile_vae(fast, cc)
    res = dict(_gpu_info(), what="SD-1.5 VAE encode, fp16, image -> moments", iters=args.iters, warmup=args.warmup,
               shapes=[])
    for b, h, w in SHAPES:
        x = (torch.rand(b, 3, h, w, device=dev, generator=torch.Generator(dev).manual_seed(1)) * 2 - 1).half()
        ms_native = _time(lambda: fast.encode(x), args.iters, args.warmup)
        plan = fast.encode._cached[("encode", b, h, w, torch.float16, torch.cuda.current_device())].plan
        static = x.clone()
        with torch.no_grad():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    eager.quant_conv(eager.encoder(static))
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                eager.quant_conv(eager.encoder(static))
        ms_eager = _time(g.replay, args.iters, args.warmup)
        with torch.no_grad():
            err = (fast.encode(x).latent_dist.parameters.float() -
                   eager.quant_conv(eager.encoder(x)).float()).abs().max().item()
        res["shapes"].append({"batch": b, "h": h, "w": w, "native_ms": ms_native, "eager_graph_ms": ms_eager,
                              "speedup": ms_eager / ms_native, "plan_tflop": plan.flops() / 1e12,
                              "native_tflops": plan.flops() / (ms_native / 1e3) / 1e12,
                              "max_abs_diff_vs_eager": err})
        del g, static, plan
        fast.encode._cached.clear()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
