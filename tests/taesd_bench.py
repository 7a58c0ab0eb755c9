"""Times the native AutoencoderTiny (TAESD) decode and encode against the same module run eagerly the way
bench.py's gpu_library_baseline runs a UNet: fp16, channels_last, cudnn.benchmark, captured in a
torch.cuda.CUDAGraph.  Sizes 512^2 and 1024^2 images, batch 1 and 4.  Also times the sfb_conv3x3_c64 launches
of each decode plan alone, as one CUDA graph, for their achieved TFLOP/s.  Device-event times; the GPU's name and
power limit are read with nvidia-smi --query-gpu.  Prints one JSON line; --json PATH also writes it to PATH.

    python tests/taesd_bench.py [--iters 20] [--json PATH]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-fast_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from oracle import taesd_oracle as to  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                          "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name()


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def graphed(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_vae
    from sfast_b200 import _lib
    torch.backends.cudnn.benchmark = True
    dt = torch.float16
    eager = to.build_taesd(seed=0, dtype=dt, device="cuda").to(memory_format=torch.channels_last)
    native = compile_vae(to.build_taesd(seed=0, dtype=dt, device="cuda"), CompilationConfig.Default())
    lib = _lib.lib()
    rows = []
    for side in (512, 1024):
        for batch in (1, 4):
            g = torch.Generator(device="cuda").manual_seed(side + batch)
            z = torch.randn(batch, 4, side // 8, side // 8, generator=g, device="cuda").to(dt)
            x = (torch.rand(batch, 3, side, side, generator=g, device="cuda") * 2 - 1).to(dt)
            zc, xc = z.to(memory_format=torch.channels_last), x.to(memory_format=torch.channels_last)
            with torch.no_grad():
                ed, ee = graphed(lambda: eager.decode(zc)), graphed(lambda: eager.encode(xc))
                t_ed, t_ee = time_ms(ed, args.iters), time_ms(ee, args.iters)
                t_nd = time_ms(lambda: native.decode(z), args.iters)
                t_ne = time_ms(lambda: native.encode(x), args.iters)
            comp = native.decode._compiled
            plan = comp._cached[("decode", batch, side // 8, side // 8, dt, z.device.index)].plan
            c64 = [op for op in plan.all_ops() if op.fn is lib.sfb_conv3x3_c64]
            t_c64 = time_ms(graphed(lambda: [op.launch(torch.cuda.current_stream().cuda_stream) for op in c64]),
                            args.iters)
            flops = sum(op.flops for op in c64)
            eplan = comp._cached[("encode", batch, side, side, dt, z.device.index)].plan
            row = dict(side=side, batch=batch, decode_native_ms=t_nd, decode_eager_graph_ms=t_ed,
                       encode_native_ms=t_ne, encode_eager_graph_ms=t_ee,
                       decode_gflop=plan.flops() / 1e9, encode_gflop=eplan.flops() / 1e9,
                       c64_decode_launches=len(c64), c64_decode_ms=t_c64, c64_tflops=flops / t_c64 / 1e9)
            rows.append(row)
            print(f"{side}^2 x{batch}: decode native {t_nd:.3f} ms vs eager graph {t_ed:.3f} ms "
                  f"({t_ed / t_nd:.2f}x) | encode native {t_ne:.3f} ms vs eager graph {t_ee:.3f} ms "
                  f"({t_ee / t_ne:.2f}x) | c64 convs of decode {t_c64:.3f} ms = {row['c64_tflops']:.0f} TFLOP/s",
                  flush=True)
    res = dict(gpu=gpu_info(), rows=rows)
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
