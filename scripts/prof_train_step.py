"""Time one training step on the device, one image: forward, backward and the optimiser step from CUDA events after a
warm-up, images/s and peak memory, in bf16 and bf16x3.  --config picks the configuration: cityscapes_r50 (UPSNet-50 at
1024x2048, the default), coco_r50 (UPSNet-50 COCO at 800x1344: fpn_with_gap, fcn_with_roi_loss) or coco_r101_dcn
(UPSNet-101 with DCN in res3-res5, COCO at 800x1344).  As a comparator, the same step composed from library ops
(tests/train_forward_oracle.py, on cuDNN: fp32 with TF32 off, and bf16 autocast) with the same discrete decisions.
Prints the card name and power limit of the run.

  python scripts/prof_train_step.py [--config cityscapes_r50] [--steps 5] [--warmup 2]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


# name: (UPSNetConfig constructor, ResNet depth, image size, dataset of the label block)
CONFIGS = {"cityscapes_r50": ("cityscapes_r50", (3, 4, 6, 3), (1024, 2048), "cityscapes"),
           "coco_r50": ("coco_r50", (3, 4, 6, 3), (800, 1344), "coco"),
           "coco_r101_dcn": ("coco_r101_dcn", (3, 4, 23, 3), (800, 1344), "coco")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--config", choices=sorted(CONFIGS), default="cityscapes_r50")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_train_step.py needs a CUDA device")
    import train_forward_oracle as TF
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    make_cfg, depth, (H, W), dataset = CONFIGS[a.config]
    cfg = getattr(UPSNetConfig, make_cfg)()
    losses = TF.COCO_LOSSES if cfg.fcn_with_roi_loss else TF.LOSSES
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    dev = torch.device("cuda", 0)
    m = synthetic_model(cfg, depth=depth, seed=0, device=dev)
    entry, lmap = TF.synthetic_entry(1, H, W, 30, num_classes=cfg.num_classes)
    np.random.seed(0)
    label = {"roidb": entry}
    label.update(U.training.RPNTargets(max_size=W).from_roidb(entry, 1.0, dev))
    label.update(U.PanopticLabels(dataset=dataset, with_roi=cfg.fcn_with_roi_loss).from_roidb(entry, lmap, (H, W), 1.0,
                                                                                             dev))
    data = {"data": TF.image(2, H, W).to(dev), "im_info": np.array([[H, W, 1.0]], np.float32)}
    opt = U.SGD(m.get_params_lr(), lr=1, momentum=0.9, weight_decay=1e-4)
    m.keep_intermediates = True
    inter = None
    for prec in ("bf16", "bf16x3"):
        U.set_precision(prec)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        times = []
        torch.cuda.reset_peak_memory_stats(dev)
        for it in range(a.warmup + a.steps):
            np.random.seed(it)
            opt.zero_grad()
            ev[0].record()
            out = m(data, label)
            ev[1].record()
            sum(out[k] for k in losses).backward()
            ev[2].record()
            opt.step(1e-6)
            ev[3].record()
            torch.cuda.synchronize()
            if it >= a.warmup:
                times.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
            inter = out["_intermediates"]
        f, b, o = np.median(np.asarray(times), 0)
        print("%s %-7s forward %.1f ms  backward %.1f ms  optimiser %.2f ms  step %.1f ms  %.2f images/s  peak %.2f GB"
              % (a.config, prec, f, b, o, f + b + o, 1000.0 / (f + b + o), torch.cuda.max_memory_allocated(dev) / 2 ** 30))
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    for name, ac in (("library fp32 (TF32 off)", None), ("library bf16 autocast", torch.bfloat16)):
        orc = TF.TrainOracle(sd, TF.trainable_names(m), depth=depth, num_classes=cfg.num_classes,
                             num_seg_classes=cfg.num_seg_classes, dconv_from=cfg.backbone_with_dconv,
                             fcn_layers=cfg.fcn_num_layers, with_gap=cfg.fpn_with_gap,
                             fcn_with_roi_loss=cfg.fcn_with_roi_loss, dtype=torch.float32, device=dev)
        times = []
        torch.cuda.reset_peak_memory_stats(dev)
        for it in range(a.warmup + a.steps):
            for p in orc.p.values():
                p.grad = None
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            with torch.autocast("cuda", dtype=ac, enabled=ac is not None):
                out = orc.forward(data["data"], label, inter)
            ev[1].record()
            sum(out[k] for k in losses).float().backward()
            ev[2].record()
            torch.cuda.synchronize()
            if it >= a.warmup:
                times.append([ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])])
        f, b = np.median(np.asarray(times), 0)
        print("%-24s forward %.1f ms  backward %.1f ms  (no optimiser)  peak %.2f GB"
              % (name, f, b, torch.cuda.max_memory_allocated(dev) / 2 ** 30))


if __name__ == "__main__":
    main()
