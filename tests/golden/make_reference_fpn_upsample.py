"""Generates tests/golden/reference_fpn_upsample.npz by EXECUTING the reference's own FPN with
upsample_method='bilinear' (network.fpn_upsample_method; build container only: /root/reference is not present on the
GPU box).
Run: python tests/golden/make_reference_fpn_upsample.py

Executed, unmodified, from /root/reference/upsnet: models/fpn.py:27-104 FPN (constructor and forward), built as
models/resnet_upsnet.py:50 builds it, with the import shims of make_reference_group_norm.py.

Three cases, fpn_feature_dim 64, on the CPU, at inputs whose P5 is 3x5 (odd, so the last row and column repeat) and
P2 24x40:
  none / none_gap / gn_gap: fpn_with_norm 'none' without and with fpn_with_gap, 'group_norm' with fpn_with_gap.
Recorded for each case <c>: <c>_param_names / <c>_param_shapes (named_parameters order) and <c>_out<i>, the five FPN
outputs P2..P6.  Inputs and parameters are not stored: tests/train_forward_oracle.py fixture_values (seeds 0-3, scale
4) and fixture_fpn_params define them, and the test makes them again.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))                    # tests/: train_forward_oracle
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))   # the repository: oracle, upsnet_b200
import make_reference_group_norm as MRG  # noqa: E402  (puts /root/reference first on sys.path)

OUT = os.path.join(HERE, "reference_fpn_upsample.npz")
CASES = (("none", "none", False), ("none_gap", "none", True), ("gn_gap", "group_norm", True))
P2_SHAPE = (24, 40)          # P5 3x5
FEATURE_DIM = 64


def inputs():
    import train_forward_oracle as TF
    h, w = P2_SHAPE
    return [TF.fixture_values(l, (1, c, h >> l, w >> l), 4.0) for l, c in enumerate((256, 512, 1024, 2048))]


def main():
    MRG.MRM._install_shims()
    MRG._stub_functions()
    import torch
    import train_forward_oracle as TF
    from upsnet.config.config import config
    out = {}
    for case, norm, with_gap in CASES:
        config.network.fpn_with_gap = with_gap
        config.network.fpn_feature_dim = FEATURE_DIM
        config.network.fpn_with_norm = norm
        config.network.fpn_upsample_method = "bilinear"
        from upsnet.models.fpn import FPN
        torch.manual_seed(0)
        # models/resnet_upsnet.py:50
        fpn = FPN(feature_dim=config.network.fpn_feature_dim, with_norm=config.network.fpn_with_norm,
                  upsample_method=config.network.fpn_upsample_method)
        shapes = [("fpn." + n, tuple(p.shape)) for n, p in fpn.named_parameters()]
        params = TF.fixture_fpn_params(shapes)
        out[case + "_param_names"] = np.array([n for n, _ in shapes])
        out[case + "_param_shapes"] = np.array([",".join(map(str, s_)) for _, s_ in shapes])
        with torch.no_grad():
            named = dict(fpn.named_parameters())
            for n, v in params.items():
                named[n[len("fpn."):]].copy_(v)
            for l, t in enumerate(fpn(*inputs())):
                out["%s_out%d" % (case, l)] = t.numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes;", {k: out[k].shape for k in out})


if __name__ == "__main__":
    main()
