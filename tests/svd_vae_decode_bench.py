"""Native temporal VAE decode vs the same AutoencoderKLTemporalDecoder run eagerly (PyTorch library kernels) under
a CUDA graph.

    python tests/svd_vae_decode_bench.py [--iters N] [--warmup W] [--chunks 8 14 25]

SVD-XT's VAE (oracle/svd_vae_oracle.py, seeded weights), fp16, 72 x 128 latents -> 576 x 1024 frames, one video
of `chunk` frames per call (StableVideoDiffusionPipeline's decode_chunk_size).  Both sides are timed with CUDA
events over N back-to-back calls after W warm-up calls: the native side is `compile_vae(m).decode(z, chunk)`
(input copy, graph replay, output clone), the eager side a captured graph of `decoder(z, chunk)`.  The two run
one after the other with the memory of the first freed: both at once do not fit at 25 frames.  "clip_ms" is
the decode of a 25-frame clip in chunks of that size (the last chunk shorter).  Prints one JSON line with the
GPU's name and power limit, read in the same process."""
import argparse
import gc
import json
import os
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (_ROOT, os.path.join(_ROOT, "stable-fast_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import svd_vae_oracle as svo  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

CLIP = 25


def _chunks(chunk):
    return [min(chunk, CLIP - i) for i in range(0, CLIP, chunk)]


def _eager_graph(m, z, nf):
    static = z.clone()
    with torch.no_grad():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            out = m.decoder(static, nf)
        torch.cuda.current_stream().wait_stream(side)
        del out
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = m.decoder(static, nf)
    return g, out


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_vae
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--chunks", type=int, nargs="+", default=[8, 14, 25])
    args = ap.parse_args(argv)
    dev = "cuda"
    cfg = svo.svd_vae_config()
    m = svo.build_svd_vae(cfg, seed=0, dtype=torch.float16, device=dev)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    m = compile_vae(m, cc)
    res = dict(_gpu_info(), what="SVD-XT VAE decode, fp16, 72x128 latents -> 576x1024 frames", iters=args.iters,
               warmup=args.warmup, chunks=[])
    z_all = (torch.randn(CLIP, 4, 72, 128, device=dev, generator=torch.Generator(dev).manual_seed(1))
             / 0.18215 * 0.2).half()
    for chunk in args.chunks:
        sizes = sorted(set(_chunks(chunk)), reverse=True)
        native, eager, row = {}, {}, {"chunk": chunk, "clip_chunks": _chunks(chunk)}
        for nf in sizes:                                   # native: plans + graphs of this clip's chunk sizes
            z = z_all[:nf]
            native[nf] = _time(lambda: m.decode(z, nf), args.iters, args.warmup)
        key = ("decode_t", chunk, chunk, 72, 128, torch.float16, torch.cuda.current_device())
        plan = m.decode._cached[key].plan
        row["plan_tflop"] = plan.flops() / 1e12
        row["plan_buffer_gb"] = sum(t.numel() * t.element_size() for t in plan._bufs.values()) / 1e9
        got = m.decode(z_all[:chunk], chunk).sample.cpu()
        del plan
        m.decode._cached.clear()
        gc.collect()
        torch.cuda.empty_cache()
        for nf in sizes:                                   # eager under a CUDA graph, same module
            g, out = _eager_graph(m, z_all[:nf], nf)
            eager[nf] = _time(g.replay, args.iters, args.warmup)
            if nf == chunk:
                g.replay()
                torch.cuda.synchronize()
                row["max_abs_diff_vs_eager"] = (got.float() - out.float().cpu()).abs().max().item()
            del g, out
            gc.collect()
            torch.cuda.empty_cache()
        row.update(native_ms=native[chunk], eager_graph_ms=eager[chunk], speedup=eager[chunk] / native[chunk],
                   native_tflops=row["plan_tflop"] / (native[chunk] / 1e3),
                   native_clip_ms=sum(native[n] for n in _chunks(chunk)),
                   eager_clip_ms=sum(eager[n] for n in _chunks(chunk)))
        res["chunks"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
