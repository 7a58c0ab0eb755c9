"""The native AnimateDiff UNet step against the oracle module run eagerly under one CUDA graph.

    python tests/animatediff_bench.py [--iters N] [--warmup W] [--rounds R] [--out DIR]

Seeded weights (oracle/animatediff_oracle.py):
  * SD-1.5 + the v1-5-2 motion geometry, 512^2 (64^2 latents), 16 frames, B = 2 (classifier-free guidance), fp16;
  * SDXL-shaped, 1024^2 (128^2 latents), 16 frames, B = 2, bf16 -- the eager leg only if it fits in memory.
Each round times N calls of the native step, then N replays of the eager graph, with CUDA events after W warm-up
calls; reports the median per-step time over R rounds, the spread (max - min) and the largest output difference.

A second, separate measurement (no graph, CUDA events around every launch of the main stream) gives the motion
modules' share of the step; a torch.profiler run (trace written under --out) gives sfb_frame_attention's kernel time
and achieved bytes/s against the data sheet's 3.35 TB/s.  Prints one JSON line with the GPU's name and power limit,
read in the same process."""
import argparse
import copy
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

from oracle import animatediff_oracle as ao  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
CASES = (("SD-1.5 v1-5-2", ao.v152_config, 64, torch.float16),
         ("SDXL", ao.sdxl_config, 128, torch.bfloat16))


def _inputs(cfg, b, f, lat, dt):
    g = torch.Generator(device="cuda").manual_seed(0)
    s = torch.randn(b, cfg.in_channels, f, lat, lat, device="cuda", generator=g).to(dt)
    e = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        n_text = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
        kw["added_cond_kwargs"] = {"text_embeds": torch.randn(b, n_text, device="cuda", generator=g).to(dt),
                                   "time_ids": torch.tensor([[8. * lat, 8 * lat, 0, 0, 8 * lat, 8 * lat]] * b,
                                                            device="cuda").to(dt)}
    return s, e, kw


class _Timed:
    """One launch of the main stream between two CUDA events."""

    def __init__(self, op):
        self.op, self.e0, self.e1 = op, torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self.name, self.fn = op.name, op.fn

    def launch(self, stream):
        self.e0.record()
        self.op.launch(stream)
        self.e1.record()


def motion_share(plan):
    """(motion-module launches' summed time, every main-stream launch's summed time) in ms, one step."""
    from sfast_b200.plan import _ForkOp, _JoinOp
    saved = plan.ops
    plan.ops = [o if isinstance(o, (_ForkOp, _JoinOp)) else _Timed(o) for o in saved]
    try:
        plan.run()
        plan.run()
        torch.cuda.synchronize()
        timed = [o for o in plan.ops if isinstance(o, _Timed)]
        tot = sum(o.e0.elapsed_time(o.e1) for o in timed)
        mot = sum(o.e0.elapsed_time(o.e1) for o in timed if ".motion_modules." in o.name)
    finally:
        plan.ops = saved
    return mot, tot


def frame_attention_profile(call, plan, out_dir, steps=3):
    """torch.profiler over `steps` native steps: sfb_frame_attention's kernel time per step and bytes/s."""
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            call()
        torch.cuda.synchronize()
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "animatediff_trace.json"))
    fa_us = sum(e.device_time_total for e in prof.key_averages() if "frame_attention_kernel" in e.key) / steps
    all_us = sum(e.device_time_total for e in prof.key_averages() if e.device_time_total > 0) / steps
    nbytes = sum(o.bytes for o in plan.all_ops() if getattr(o.fn, "__name__", None) == "sfb_frame_attention")
    return {"frame_attention_ms_per_step": fa_us / 1000, "kernels_ms_per_step": all_us / 1000,
            "frame_attention_bytes_per_step": nbytes,
            "frame_attention_bytes_per_s": nbytes / (fa_us * 1e-6) if fa_us else None,
            "frame_attention_share_of_3_35_TBps": nbytes / (fa_us * 1e-6) / HBM_BYTES_PER_S if fa_us else None}


def run_case(name, cfgf, lat, dt, args, b=2, f=16):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    cfg = cfgf()
    eager = ao.build_unet(cfg, seed=1, dtype=dt, device="cuda")
    fast = compile_unet(copy.deepcopy(eager), cc)
    s, e, kw = _inputs(cfg, b, f, lat, dt)
    t = torch.tensor(500, device="cuda")
    native = fast(s, t, e, **kw).sample
    case = {"model": name, "dtype": str(dt).replace("torch.", ""), "videos": b, "frames": f, "latent": lat,
            "first_call_s": fast.forward._compiled.first_call_s}
    graph = None
    try:
        with torch.no_grad():
            for _ in range(2):
                eager(s, t, e, **kw)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                ref = eager(s, t, e, **kw).sample
        graph.replay()
        torch.cuda.synchronize()
        case["max_abs_diff_vs_eager"] = (native.float() - ref.float()).abs().max().item()
        case["max_abs_eager"] = ref.float().abs().max().item()
    except torch.cuda.OutOfMemoryError as exc:
        graph = None
        case["eager"] = f"not measured: out of memory ({str(exc).splitlines()[0]})"
    torch.cuda.empty_cache()
    nat, eag = [], []
    for _ in range(args.rounds):
        nat.append(_time(lambda: fast(s, t, e, **kw), args.iters, args.warmup))
        if graph is not None:
            eag.append(_time(graph.replay, args.iters, args.warmup))
    case.update(native_step_ms=statistics.median(nat), native_spread_ms=max(nat) - min(nat))
    if eag:
        case.update(eager_graph_step_ms=statistics.median(eag), eager_spread_ms=max(eag) - min(eag),
                    speedup=statistics.median(eag) / statistics.median(nat))
    del graph
    torch.cuda.empty_cache()
    plan = next(iter(fast.forward._cached.values())).plan
    mot, tot = motion_share(plan)
    case.update(motion_ms_per_step_event_timed=mot, step_ms_event_timed=tot, motion_share=mot / tot)
    if name.startswith("SD-1.5"):
        case.update(frame_attention_profile(lambda: fast(s, t, e, **kw), plan, args.out))
    return case


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args(argv)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    res = dict(_gpu_info(), what="AnimateDiff UNet step: native vs the oracle module eager under one CUDA graph",
               iters=args.iters, warmup=args.warmup, rounds=args.rounds, cases=[])
    for name, cfgf, lat, dt in CASES:
        try:
            res["cases"].append(run_case(name, cfgf, lat, dt, args))
        except torch.cuda.OutOfMemoryError as exc:
            res["cases"].append({"model": name, "error": f"out of memory: {str(exc).splitlines()[0]}"})
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(os.path.join(args.out, "animatediff_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
