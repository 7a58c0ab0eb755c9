"""Native T2I-Adapter vs the same adapter run eagerly (PyTorch library kernels) under a CUDA graph, and the UNet step
with and without the adapter's residuals.

    python tests/t2i_adapter_bench.py [--iters N] [--warmup W]

Seeded weights (oracle/t2i_adapter_oracle.py, oracle/unet_oracle.py).  Timed with CUDA events over N back-to-back
calls after W warm-up calls:
  * adapter: SD-1.5's full_adapter at 512^2 in fp16 and SDXL's full_adapter_xl at 1024^2 in bf16, B = 1 (the adapter
    runs once per pipeline call, on the un-duplicated image):
      native_ms: `compile_adapter(m)(x)` (input copy, graph replay, feature clones);
      eager_graph_ms: the oracle module in the same dtype, captured as one CUDA graph;
      max_rel_diff_vs_eager: the largest feature's max |native - eager| / max |eager|;
  * UNet step at B = 2 (one image with classifier-free guidance): SD-1.5 at 64^2 latents in fp16, SDXL at 128^2 in
    bf16; plain_step_ms without residuals, adapter_step_ms with the adapter's features as
    down_intrablock_additional_residuals (4 in-place adds per step).
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

from oracle import t2i_adapter_oracle as to  # noqa: E402
from oracle import unet_oracle as uo  # noqa: E402
from vae_encode_bench import _gpu_info, _time  # noqa: E402

CASES = (("SD-1.5", to.sd_config, uo.sd15_config, 512, torch.float16),
         ("SDXL", to.sdxl_config, uo.sdxl_config, 1024, torch.bfloat16))


def _unet_kw(cfg, b, lat, dt, g):
    if cfg.addition_embed_type != "text_time":
        return {}
    size = 8 * lat
    return {"added_cond_kwargs": dict(text_embeds=torch.randn(b, 1280, device="cuda", generator=g).to(dt),
                                      time_ids=torch.tensor([[size, size, 0, 0, size, size]] * b, device="cuda",
                                                            dtype=torch.float32))}


def main(argv=None):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_adapter, compile_unet
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    res = dict(_gpu_info(), what="T2I-Adapter call (B=1) native vs eager under a CUDA graph; UNet step (B=2) with "
               "and without the adapter residuals", iters=args.iters, warmup=args.warmup, cases=[])
    for name, a_cfg_f, u_cfg_f, size, dt in CASES:
        a_cfg, u_cfg = a_cfg_f(), u_cfg_f()
        g = torch.Generator(device="cuda").manual_seed(0)
        img = torch.rand(1, a_cfg.in_channels, size, size, device="cuda", generator=g).to(dt)
        eager = to.build_adapter(a_cfg, seed=0, dtype=dt, device="cuda")
        native = compile_adapter(to.build_adapter(a_cfg, seed=0, dtype=dt, device="cuda"), cc)
        ms_native = _time(lambda: native(img), args.iters, args.warmup)
        feats = native(img)
        with torch.no_grad():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    eager(img)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                eager_feats = eager(img)
            ms_eager = _time(graph.replay, args.iters, args.warmup)
            graph.replay()
            torch.cuda.synchronize()
            diff = max(((f.float() - e.float()).abs().max() / e.float().abs().max()).item()
                       for f, e in zip(feats, eager_feats))
        del graph, eager, eager_feats
        torch.cuda.empty_cache()

        lat, b = size // 8, 2
        unet = compile_unet(uo.build_unet(u_cfg, seed=1, dtype=dt, device="cuda"), cc)
        sample = torch.randn(b, 4, lat, lat, device="cuda", generator=g).to(dt)
        ehs = torch.randn(b, 77, u_cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
        t = torch.tensor(500, device="cuda")
        kw = _unet_kw(u_cfg, b, lat, dt, g)
        residuals = [torch.cat([f * 0.8] * b) for f in feats]
        ms_plain = _time(lambda: unet(sample, t, ehs, **kw), args.iters, args.warmup)
        ms_adapter = _time(lambda: unet(sample, t, ehs, down_intrablock_additional_residuals=residuals, **kw),
                           args.iters, args.warmup)
        res["cases"].append({"model": name, "dtype": str(dt).replace("torch.", ""), "image": size,
                             "adapter_native_ms": ms_native, "adapter_eager_graph_ms": ms_eager,
                             "adapter_speedup": ms_eager / ms_native, "max_rel_diff_vs_eager": diff,
                             "unet_batch": b, "latent": lat, "plain_step_ms": ms_plain,
                             "adapter_step_ms": ms_adapter, "adapter_step_overhead_ms": ms_adapter - ms_plain})
        del native, unet, feats, residuals
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
