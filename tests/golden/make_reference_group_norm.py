"""Generates tests/golden/reference_group_norm.npz by EXECUTING the reference's own head constructors and its
get_params_lr (build container only: /root/reference is not present on the GPU box).
Run: python tests/golden/make_reference_group_norm.py

Executed, unmodified, from /root/reference/upsnet:
  models/fpn.py:27-104 FPN (constructor and forward), models/rpn.py:27-56 RPN, models/rcnn.py:36-87 MaskBranch and
  :91-111 RCNN, models/fcn.py:31-60 FCNSubNet and :77-86 FCNHead (constructors),
  models/resnet_upsnet.py:260-285 get_params_lr with models/resnet.py:31-51 get_params (taken out of their files by
  ast, because resnet_upsnet.py imports the un-built CUDA extensions).
The heads are built with the arguments models/resnet_upsnet.py:50-60 passes (the RPN without with_norm).

Recorded for each norm option ('none', 'group_norm' on all four keys):
  <opt>_keys / <opt>_shapes: the head state_dict (fpn, rpn, rcnn, mask_branch, fcn_head) key and shape list;
  <opt>_group<i>: the parameter names of get_params_lr group i (13 groups; res3-res5 are not built here, so their
  groups are empty);
  gn_fpn_out<i> / gn_rpn_<k>: the group_norm FPN (with fpn_gap, fpn_feature_dim 64) on 8x16 inputs and the RPN on
  its P2, run on the CPU; inputs and parameters (gn_param_names / gn_param_shapes, in named_parameters order) are
  not stored but defined by tests/train_forward_oracle.py fixture_values / fixture_fpn_params.

Import shims (nothing inside the executed code is changed): those of make_reference_modules.py, plus stand-ins for
the ROIAlign / deformable-conv autograd Functions (CUDA extensions; the constructors do not call them).
"""
import ast
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))                    # tests/: train_forward_oracle
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))   # the repository: oracle, upsnet_b200
import make_reference_modules as MRM  # noqa: E402  (puts /root/reference first on sys.path)

OUT = os.path.join(HERE, "reference_group_norm.npz")
NORM_KEYS = ("fpn_with_norm", "rpn_with_norm", "rcnn_with_norm", "fcn_with_norm")


def _stub_functions():
    for name, attrs in (("upsnet.operators.functions.roialign", ("RoIAlignFunction",)),
                        ("upsnet.operators.functions.deform_conv", ("DeformConvFunction",))):
        m = types.ModuleType(name)
        for a in attrs:
            setattr(m, a, type(a, (), {}))
        sys.modules[name] = m
    # upsnet/models/__init__.py imports resnet_upsnet.py and with it the training operators (pycocotools, CUDA):
    # the head files are loaded as submodules of a bare package instead
    import upsnet  # noqa: F401
    pkg = types.ModuleType("upsnet.models")
    pkg.__path__ = ["/root/reference/upsnet/models"]
    sys.modules["upsnet.models"] = pkg


def _extract(path, names):
    """The top-level functions `names` of a reference file, compiled on their own."""
    tree = ast.parse(open(path).read())
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    body += [f for n in tree.body if isinstance(n, ast.ClassDef) for f in n.body
             if isinstance(f, ast.FunctionDef) and f.name in names]
    return ast.Module(body=body, type_ignores=[])


def build_heads(norm, with_gap, feature_dim=256):
    import torch.nn as nn
    from upsnet.config.config import config
    config.dataset.num_classes, config.dataset.num_seg_classes = 9, 19
    config.network.fpn_with_gap = with_gap
    config.network.fpn_feature_dim = feature_dim
    for k in NORM_KEYS:
        config.network[k] = norm
    from upsnet.models.fpn import FPN
    from upsnet.models.rpn import RPN
    from upsnet.models.rcnn import RCNN, MaskBranch
    from upsnet.models.fcn import FCNHead
    heads = nn.Module()
    # models/resnet_upsnet.py:50-60
    heads.fpn = FPN(feature_dim=config.network.fpn_feature_dim, with_norm=config.network.fpn_with_norm,
                    upsample_method=config.network.fpn_upsample_method)
    heads.rpn = RPN(num_anchors=config.network.num_anchors, input_dim=config.network.fpn_feature_dim)
    heads.rcnn = RCNN(9, 9, dim_in=config.network.fpn_feature_dim, with_norm=config.network.rcnn_with_norm)
    heads.mask_branch = MaskBranch(9, dim_in=config.network.fpn_feature_dim, with_norm=config.network.rcnn_with_norm)
    heads.fcn_head = FCNHead(config.network.fpn_feature_dim, 19, num_layers=config.network.fcn_num_layers,
                             with_norm=config.network.fcn_with_norm, upsample_rate=4,
                             with_roi_loss=config.train.fcn_with_roi_loss)
    return heads


def param_groups(heads):
    import torch.nn as nn
    from upsnet.config.config import config
    ns = {"nn": nn, "config": config}
    exec(compile(_extract("/root/reference/upsnet/models/resnet.py", {"get_params"}), "resnet.py", "exec"), ns)
    exec(compile(_extract("/root/reference/upsnet/models/resnet_upsnet.py", {"get_params_lr"}), "resnet_upsnet.py",
                 "exec"), ns)
    names = {id(p): n for n, p in heads.named_parameters()}
    return [[names[id(p)] for p in g["params"]] for g in ns["get_params_lr"](heads)]


def main():
    MRM._install_shims()
    _stub_functions()
    import torch
    out = {}
    for norm in ("none", "group_norm"):
        torch.manual_seed(0)
        heads = build_heads(norm, with_gap=False)
        sd = heads.state_dict()
        out[norm + "_keys"] = np.array(list(sd.keys()))
        out[norm + "_shapes"] = np.array([",".join(map(str, v.shape)) for v in sd.values()])
        for i, g in enumerate(param_groups(heads)):
            out["%s_group%d" % (norm, i)] = np.array(g, dtype=str)
    # the group_norm FPN (with the context vector) and RPN, executed at a small size on inputs and parameters that
    # train_forward_oracle.fixture_values defines, so that only their names, shapes and the outputs are stored
    import train_forward_oracle as TF
    torch.manual_seed(1)
    heads = build_heads("group_norm", with_gap=True, feature_dim=64)      # 64 channels: a small fixture
    shapes = [(n, tuple(p.shape)) for n, p in heads.named_parameters() if n.startswith(("fpn.", "rpn."))]
    params = TF.fixture_fpn_params(shapes)
    out["gn_param_names"] = np.array([n for n, _ in shapes])
    out["gn_param_shapes"] = np.array([",".join(map(str, s_)) for _, s_ in shapes])
    with torch.no_grad():
        named = dict(heads.named_parameters())
        for n, v in params.items():
            named[n].copy_(v)
        ins = [TF.fixture_values(l, (1, c, 8 >> l, 16 >> l), 4.0) for l, c in enumerate((256, 512, 1024, 2048))]
        fpn = heads.fpn(*ins)
        for l, t in enumerate(fpn):
            out["gn_fpn_out%d" % l] = t.numpy()
        for k, t in zip(("cls_score", "bbox_pred", "cls_prob"), heads.rpn(fpn[0])):
            out["gn_rpn_" + k] = t.numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes;", {k: out[k].shape for k in out})


if __name__ == "__main__":
    main()
