"""LoRA on the native UNet: step time without and with a merged rank-64 adapter on every weight, the switch
latency after set_adapters changes a weight (and its split between sfb_lora_merge and re-packing), and the
per-call host cost of the adapter-state check.  One JSON line per setup; the card name and power limit are read
in the same run.

    python tests/lora_bench.py [--setups sd15,sdxl] [--steps 50] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-fast_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import torch  # noqa: E402

from oracle import lora_oracle as lo  # noqa: E402
from oracle import unet_oracle as uo  # noqa: E402
from sfast_b200 import ops  # noqa: E402

SETUPS = {"sd15": (uo.sd15_config, 512, torch.float16), "sdxl": (uo.sdxl_config, 1024, torch.bfloat16)}


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def _compile(m):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    return compile_unet(m, cc)


def _step_ms(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def _wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def run(name, steps, rounds):
    cfg_fn, px, dt = SETUPS[name]
    cfg = cfg_fn()
    h = px // 8
    dev = "cuda:0"
    plain = _compile(uo.build_unet(cfg, seed=0, dtype=dt, device=dev))
    adapted = _compile(lo.inject_adapter(uo.build_unet(cfg, seed=0, dtype=dt, device=dev), "a", "all", r=64,
                                         lora_alpha=64, seed=1))
    g = torch.Generator(device=dev).manual_seed(0)
    s = torch.randn(2, 4, h, h, device=dev, generator=g).to(dt)
    e = torch.randn(2, 77, cfg.cross_attention_dim, device=dev, generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        kw = dict(added_cond_kwargs=dict(text_embeds=torch.randn(2, 1280, device=dev, generator=g).to(dt),
                                         time_ids=torch.tensor([[px, px, 0, 0, px, px]] * 2, device=dev, dtype=dt)))
    t = torch.tensor(500, device=dev)
    calls = {"none": lambda: plain(s, t, e, **kw), "merged": lambda: adapted(s, t, e, **kw)}
    for fn in calls.values():
        for _ in range(5):
            fn()
    times = {k: [] for k in calls}
    for _ in range(rounds):  # alternate, one process
        for k, fn in calls.items():
            times[k].append(_step_ms(fn, steps))

    # switch latency: the first call after set_adapters changes a weight, minus a steady call
    compiled = adapted.forward._compiled
    steady = min(_wall_ms(calls["merged"]) for _ in range(5))
    switch = []
    for i in range(rounds):
        lo.set_adapters(adapted, "a", 0.5 + 0.25 * i)
        switch.append(_wall_ms(calls["merged"]) - steady)

    # the merge alone: every adapted layer's sfb_lora_merge, CUDA events around the launches
    layers = list(compiled._lora.layers.values())
    args = []
    nbytes = 0
    for layer in layers:
        w = layer.base_layer.weight.detach()
        a, b = layer.lora_A["a"].weight.detach(), layer.lora_B["a"].weight.detach()
        args.append((w.reshape(w.shape[0], -1), [(a.reshape(a.shape[0], -1), b.reshape(w.shape[0], -1), 0.5)]))
        nbytes += w.element_size() * w.numel() * 2 + a.element_size() * (a.numel() + b.numel())
    for wm, ad in args:
        ops.lora_merge(wm, ad, dt)
    merge_ms = _step_ms(lambda: [ops.lora_merge(wm, ad, dt) for wm, ad in args], 3)

    # host cost of the per-call adapter-state check (no change), with and without LoRA layers
    def check_us(c, n=200):
        t0 = time.perf_counter()
        for _ in range(n):
            c._poll_lora(1.0)
        return (time.perf_counter() - t0) / n * 1e6

    out = dict(setup=name, card=_card(), batch=2, px=px, dtype=str(dt).replace("torch.", ""), rank=64,
               adapted_layers=len(layers), step_ms_no_adapter=times["none"], step_ms_merged_adapter=times["merged"],
               switch_latency_ms=switch, merge_all_layers_ms=merge_ms,
               merge_gbps=nbytes / merge_ms / 1e6, merge_share_of_3350_gbps=nbytes / merge_ms / 1e6 / 3350,
               repack_and_other_ms=[x - merge_ms for x in switch],
               check_us_with_adapter=check_us(compiled), check_us_no_adapter=check_us(plain.forward._compiled))
    print(json.dumps(out), flush=True)
    del plain, adapted
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--setups", default="sd15,sdxl")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lora_bench.py needs an H100")
    for name in a.setups.split(","):
        run(name, a.steps, a.rounds)


if __name__ == "__main__":
    main()
