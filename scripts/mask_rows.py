"""Prints, for the four synthetic images bench.py rotates, how many rows of the static mask branch are live work:
n1 detections, n2 panoptic candidates, and u = n1 + the candidates whose box (all five floats, bit for bit) matches
no detection.  The static buffers hold 2 x 128 rows; the rest is padding.

    python scripts/mask_rows.py [--workload cityscapes|coco]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import upsnet_b200 as U  # noqa: E402
from upsnet_b200.model import UPSNetConfig  # noqa: E402
from upsnet_b200.synthetic import synthetic_input, synthetic_model  # noqa: E402


def distinct_rows(b1, n1, b2, n2):
    d = b1[:n1].contiguous().view(torch.int32)
    c = b2[:n2].contiguous().view(torch.int32)
    dup = (c[:, None, :] == d[None, :, :]).all(-1).any(-1) if n1 else torch.zeros(n2, dtype=torch.bool, device=c.device)
    return n1 + int((~dup).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cityscapes", choices=["cityscapes", "coco"])
    args = ap.parse_args()
    U.set_precision("bf16x3")
    dev = torch.device("cuda", 0)
    if args.workload == "coco":
        H, W, seeds = 800, 1344, [700 + s for s in range(4)]
        model = synthetic_model(UPSNetConfig.coco_r101_dcn(), depth=(3, 4, 23, 3), seed=0, device=dev)
    else:
        H, W, seeds = 1024, 2048, list(range(4))
        model = synthetic_model(UPSNetConfig.cityscapes_r50(), seed=0, device=dev)
    im_info = synthetic_input(8, 8)["im_info"]
    im_info[0, :2] = (H, W)
    model.prepare()
    for s in seeds:
        x = synthetic_input(H, W, seed=s)["data"].to(dev)
        out, _ = model._run_static(x, im_info[0])
        n1, n2, k = (int(v) for v in out["counts"].tolist())
        u = distinct_rows(out["pred_boxes"], n1, out["p_boxes"], n2)
        print("%s seed %d: n1 %d  n2 %d  kept %d  distinct rows u %d  (of %d static rows)"
              % (args.workload, s, n1, n2, k, u, out["pred_boxes"].shape[0] + out["p_boxes"].shape[0]))


if __name__ == "__main__":
    main()
