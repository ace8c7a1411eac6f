"""GroupNorm heads (network.*_with_norm) without a GPU: the configuration keys, the module tree and parameter groups
against the reference's own constructors and get_params_lr (tests/golden/make_reference_group_norm.py), and the
literal model's group_norm FPN and RPN against the reference-executed outputs."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_forward_oracle as TF  # noqa: E402

from oracle.literal_model import LiteralUPSNet  # noqa: E402
from upsnet_b200._lib import UpsnetError  # noqa: E402
from upsnet_b200.model import UPSNetConfig, resnet_upsnet  # noqa: E402

FIX = np.load(os.path.join(HERE, "golden", "reference_group_norm.npz"))
NORM_KEYS = ("fpn_with_norm", "rpn_with_norm", "rcnn_with_norm", "fcn_with_norm")
HEADS = ("fpn.", "rpn.", "rcnn.", "mask_branch.", "fcn_head.")


def _model(norm, **kw):
    return resnet_upsnet([1, 1, 1, 1], UPSNetConfig(**dict({k: norm for k in NORM_KEYS}, **kw)))


def test_from_reference_config_reads_the_norm_keys():
    config = {"network": {"fpn_with_norm": "group_norm", "rpn_with_norm": "none", "rcnn_with_norm": "group_norm",
                          "fcn_with_norm": "none"}}
    cfg = UPSNetConfig.from_reference_config(config)
    assert (cfg.fpn_with_norm, cfg.rpn_with_norm, cfg.rcnn_with_norm, cfg.fcn_with_norm) == \
        ("group_norm", "none", "group_norm", "none")
    cfg = UPSNetConfig.from_reference_config({"network": {}})
    assert all(getattr(cfg, k) == "none" for k in NORM_KEYS)


@pytest.mark.parametrize("key", ["fpn_with_norm", "rcnn_with_norm", "fcn_with_norm"])
def test_batch_norm_is_refused_naming_the_key(key):
    with pytest.raises(UpsnetError, match=key):
        resnet_upsnet([1, 1, 1, 1], UPSNetConfig(**{key: "batch_norm"}))
    with pytest.raises(UpsnetError, match=key):
        resnet_upsnet([1, 1, 1, 1], UPSNetConfig(**{key: "sync_bn"}))


def test_rpn_norm_key_is_unused_as_in_the_reference():
    m = _model("none", rpn_with_norm="group_norm")
    assert list(m.rpn.state_dict()) == list(_model("none").rpn.state_dict())


def test_none_builds_the_default_tree():
    a, b = resnet_upsnet([1, 1, 1, 1], UPSNetConfig()), _model("none")
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(sa[k].shape == sb[k].shape for k in sa)
    assert not any(isinstance(m, torch.nn.GroupNorm) for m in b.modules())


@pytest.mark.parametrize("norm", ["none", "group_norm"])
def test_state_dict_and_param_groups_match_the_reference(norm):
    m = _model(norm, fcn_num_layers=3)        # upsnet/config/config.py's default, which the fixture's heads use
    sd = m.state_dict()
    heads = [(k, ",".join(map(str, v.shape))) for k, v in sd.items() if k.startswith(HEADS)]
    assert [k for k, _ in heads] == list(FIX[norm + "_keys"])
    assert [s for _, s in heads] == list(FIX[norm + "_shapes"])
    names = {id(p): n for n, p in m.named_parameters()}
    groups = m.get_params_lr()
    assert len(groups) == 13
    for i, g in enumerate(groups):
        got = [names[id(p)] for p in g["params"] if names[id(p)].startswith(HEADS)]
        assert got == list(FIX["%s_group%d" % (norm, i)]), i
    assert [(g["lr"], g.get("weight_decay")) for g in groups][:3] == [(1, 0), (1, None), (2, 0)]


def test_reference_style_load_accepts_a_group_norm_checkpoint():
    import warnings
    src, dst = _model("group_norm"), _model("group_norm")
    with torch.no_grad():
        for p in src.parameters():
            p.add_(0.5)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        dst.load_state_dict({"module." + k: v for k, v in src.state_dict().items()}, resume=True)
    assert all(torch.equal(a, b) for a, b in zip(src.state_dict().values(), dst.state_dict().values()))


def test_literal_group_norm_fpn_and_rpn_match_the_reference():
    shapes = [(n, tuple(int(v) for v in s.split(","))) for n, s in zip(FIX["gn_param_names"], FIX["gn_param_shapes"])]
    lit = LiteralUPSNet(TF.fixture_fpn_params(shapes), with_gap=True, dtype=torch.float64)
    ins = [TF.fixture_values(l, (1, c, 8 >> l, 16 >> l), 4.0).double() for l, c in enumerate((256, 512, 1024, 2048))]
    with torch.no_grad():
        out = lit.fpn(*ins)
        rpn = lit.rpn(out[0])
    for l, t in enumerate(out):
        want = torch.from_numpy(FIX["gn_fpn_out%d" % l]).double()
        assert float((t - want).abs().max()) <= 1e-4 * float(want.abs().max()), l
    for k, t in zip(("cls_score", "bbox_pred", "cls_prob"), rpn):
        want = torch.from_numpy(FIX["gn_rpn_" + k]).double()
        assert float((t - want).abs().max()) <= 1e-4 * max(1.0, float(want.abs().max())), k
