"""Cost of the FPN's bilinear top-down path (network.fpn_upsample_method = 'bilinear'):
python scripts/prof_fpn_upsample.py [iters]

1. The up-sampling kernel (ops.upsample2_bilinear, pair / bf16 / fp32 NHWC) and its adjoint
   (training.upsample2_bilinear_adjoint, fp32 NHWC) at the P3->P2, P4->P3 and P5->P4 shapes of 1024x2048 and 800x1344
   (256 channels): CUDA-event time per call over `iters` calls, the bytes each must move (the coarse map read once and
   the 4x larger fine map written, or the reverse), GB/s and the fraction of the H100 SXM's 3.35 TB/s.
2. Engine images/s (the static forward replayed from its CUDA graph, host clock around `iters` replays ending in a
   synchronise), 'nearest' against 'bilinear', for cityscapes_r50 and coco_r50, bf16x3 and bf16, fpn_with_norm 'none'
   and 'group_norm'; the two methods run alternately, `rounds` times each, on models with the same weights.
3. One training step (forward(data, label) + backward, bf16x3) of cityscapes_r50 at 512x1024 for each method, the two
   methods alternated `rounds` times.
The card, its power limit and clocks are read in the same run."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import upsnet_b200 as U  # noqa: E402
from prof_group_norm import events_ms  # noqa: E402
from prof_rpn_targets import card  # noqa: E402
from upsnet_b200 import operators as ops, training  # noqa: E402
from upsnet_b200.model import UPSNetConfig  # noqa: E402
from upsnet_b200.synthetic import synthetic_input, synthetic_model  # noqa: E402

HBM = 3.35e12
DEV = torch.device("cuda", 0)
SIZES = (("1024x2048", (1024, 2048)), ("800x1344", (800, 1344)))


def kernel_table(iters):
    rows = []
    g = torch.Generator().manual_seed(0)
    for size, (H, W) in SIZES:
        for step, l in (("P3->P2", 3), ("P4->P3", 4), ("P5->P4", 5)):
            h, w = -(-H // 2 ** l), -(-W // 2 ** l)
            x32 = torch.randn(1, 256, h, w, generator=g).to(DEV)
            for fmt in ("pair", "bf16", "f32"):
                if fmt == "pair":
                    x, esize = ops.Pair.from_float(x32), 4
                else:
                    x = x32.to(torch.bfloat16 if fmt == "bf16" else torch.float32).contiguous(
                        memory_format=torch.channels_last)
                    esize = 2 if fmt == "bf16" else 4
                nbytes = 5 * x32.numel() * esize
                ms = events_ms(lambda: ops.upsample2_bilinear(x), iters)      # noqa: B023
                rows.append({"size": size, "step": step, "kernel": "forward " + fmt, "coarse": [256, h, w],
                             "ms": round(ms, 4), "bytes_mb": round(nbytes / 1e6, 2), "gb_s": round(nbytes / ms / 1e6, 1),
                             "hbm_fraction": round(nbytes / ms / 1e-3 / HBM, 3)})
            dy = torch.randn(1, 256, 2 * h, 2 * w, generator=g).to(DEV).contiguous(memory_format=torch.channels_last)
            nbytes = 5 * x32.numel() * 4
            ms = events_ms(lambda: training.upsample2_bilinear_adjoint(dy), iters)  # noqa: B023
            rows.append({"size": size, "step": step, "kernel": "adjoint f32", "coarse": [256, h, w],
                         "ms": round(ms, 4), "bytes_mb": round(nbytes / 1e6, 2), "gb_s": round(nbytes / ms / 1e6, 1),
                         "hbm_fraction": round(nbytes / ms / 1e-3 / HBM, 3)})
    return rows


def _cfg(name, norm, method):
    cfg = getattr(UPSNetConfig, name)()
    cfg.fpn_with_norm = norm
    cfg.fpn_upsample_method = method
    return cfg


def engine(iters, rounds=3):
    out = {}
    for name, (H, W) in (("cityscapes_r50", (1024, 2048)), ("coco_r50", (800, 1344))):
        inp = synthetic_input(H, W, seed=1, device=DEV)
        for norm in ("none", "group_norm"):
            models = {m: synthetic_model(_cfg(name, norm, m), seed=0, device=DEV) for m in ("nearest", "bilinear")}
            for prec in ("bf16x3", "bf16"):
                U.set_precision(prec)
                runs = {m: [] for m in models}
                with torch.no_grad():
                    for m in models.values():
                        m._run_static(inp["data"], inp["im_info"][0])
                    torch.cuda.synchronize()
                    for _ in range(rounds):
                        for method, m in models.items():
                            t0 = time.perf_counter()
                            for _ in range(iters):
                                m._run_static(inp["data"], inp["im_info"][0])
                            torch.cuda.synchronize()
                            runs[method].append(round(iters / (time.perf_counter() - t0), 2))
                for method in models:
                    out["%s %s %s %s" % (name, norm, prec, method)] = {"images_s": max(runs[method]),
                                                                      "runs": runs[method]}
            del models
            torch.cuda.empty_cache()
    U.set_precision("fp32")
    return out


def train_step(iters, rounds=3):
    import train_forward_oracle as TF
    from upsnet_b200.training import PanopticLabels, RPNTargets
    H, W = 512, 1024
    entry, lmap = TF.synthetic_entry(1, H, W, 8)
    label = {"roidb": entry}
    np.random.seed(0)
    label.update(RPNTargets(max_size=max(H, W)).from_roidb(entry, 1.0, DEV))
    label.update(PanopticLabels(dataset="cityscapes").from_roidb(entry, lmap, (H, W), 1.0, DEV))
    data = {"data": TF.image(2, H, W).to(DEV), "im_info": np.array([[H, W, 1.0]], np.float32)}
    models = {m: synthetic_model(_cfg("cityscapes_r50", "none", m), seed=0, device=DEV) for m in ("nearest", "bilinear")}
    U.set_precision("bf16x3")

    def step(m):
        m.zero_grad(set_to_none=True)
        np.random.seed(5)
        o = m(data, label)
        sum(o[k] for k in TF.LOSSES).backward()
    for m in models.values():
        step(m)
    torch.cuda.synchronize()
    runs = {m: [] for m in models}
    for _ in range(rounds):
        for method, m in models.items():
            t0 = time.perf_counter()
            for _ in range(iters):
                step(m)
            torch.cuda.synchronize()
            runs[method].append(round((time.perf_counter() - t0) / iters * 1e3, 2))
    U.set_precision("fp32")
    return {"cityscapes_r50 512x1024 none %s step_ms" % m: {"best": min(r), "runs": r} for m, r in runs.items()}


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    res = {"card": card()}
    res["kernels"] = kernel_table(iters)
    res["engine_images_s"] = engine(iters)
    res["train_step"] = train_step(max(5, iters // 3))
    res["card_after"] = card()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
