"""network.fpn_upsample_method without a GPU: the configuration key, the module tree and parameter groups of both
methods, and the literal model's bilinear FPN against the reference's own FPN executed with upsample_method='bilinear'
(tests/golden/make_reference_fpn_upsample.py), and that the nearest literal model differs from it."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_forward_oracle as TF  # noqa: E402

from fpn_upsample_oracle import BilinearLiteralUPSNet  # noqa: E402
from oracle.literal_model import LiteralUPSNet  # noqa: E402
from upsnet_b200._lib import UpsnetError  # noqa: E402
from upsnet_b200.model import UPSNetConfig, resnet_upsnet  # noqa: E402

FIX = np.load(os.path.join(HERE, "golden", "reference_fpn_upsample.npz"))
CASES = {"none": ("none", False), "none_gap": ("none", True), "gn_gap": ("group_norm", True)}
P2_SHAPE = (24, 40)


def test_from_reference_config_reads_the_upsample_key():
    cfg = UPSNetConfig.from_reference_config({"network": {"fpn_upsample_method": "bilinear"}})
    assert cfg.fpn_upsample_method == "bilinear"
    assert UPSNetConfig.from_reference_config({"network": {}}).fpn_upsample_method == "nearest"
    assert UPSNetConfig().fpn_upsample_method == "nearest"
    m = resnet_upsnet([1, 1, 1, 1], UPSNetConfig(fpn_upsample_method="bilinear"))
    assert m.fpn.upsample_method == "bilinear"


@pytest.mark.parametrize("value", ["bicubic", "Bilinear", "area", ""])
def test_other_upsample_methods_are_refused_naming_the_key(value):
    with pytest.raises(UpsnetError, match="fpn_upsample_method"):
        resnet_upsnet([1, 1, 1, 1], UPSNetConfig(fpn_upsample_method=value))
    cfg = UPSNetConfig.from_reference_config({"network": {"fpn_upsample_method": value}})
    with pytest.raises(UpsnetError, match="fpn_upsample_method"):
        resnet_upsnet([1, 1, 1, 1], cfg)


@pytest.mark.parametrize("norm", ["none", "group_norm"])
@pytest.mark.parametrize("with_gap", [False, True])
def test_keys_shapes_and_param_groups_do_not_depend_on_the_method(norm, with_gap):
    def build(method):
        torch.manual_seed(0)
        return resnet_upsnet([1, 1, 1, 1], UPSNetConfig(fpn_with_norm=norm, fpn_with_gap=with_gap,
                                                         fpn_upsample_method=method))
    a, b = build("nearest"), build("bilinear")
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(sa[k].shape == sb[k].shape for k in sa)
    na = {id(p): n for n, p in a.named_parameters()}
    nb = {id(p): n for n, p in b.named_parameters()}
    ga, gb = a.get_params_lr(), b.get_params_lr()
    assert len(ga) == len(gb)
    for x, y in zip(ga, gb):
        assert [na[id(p)] for p in x["params"]] == [nb[id(p)] for p in y["params"]]
        assert {k: v for k, v in x.items() if k != "params"} == {k: v for k, v in y.items() if k != "params"}


def _inputs():
    h, w = P2_SHAPE
    return [TF.fixture_values(l, (1, c, h >> l, w >> l), 4.0).double() for l, c in enumerate((256, 512, 1024, 2048))]


@pytest.mark.parametrize("case", list(CASES))
def test_literal_bilinear_fpn_matches_the_reference(case):
    norm, with_gap = CASES[case]
    shapes = [(n, tuple(int(v) for v in s.split(","))) for n, s in
              zip(FIX[case + "_param_names"], FIX[case + "_param_shapes"])]
    assert any(".1.weight" in n for n, _ in shapes) == (norm == "group_norm")
    assert any("fpn_gap" in n for n, _ in shapes) == with_gap
    lit = BilinearLiteralUPSNet(TF.fixture_fpn_params(shapes), with_gap=with_gap, dtype=torch.float64)
    near = LiteralUPSNet(TF.fixture_fpn_params(shapes), with_gap=with_gap, dtype=torch.float64)
    with torch.no_grad():
        out = lit.fpn(*_inputs())
        nearest = near.fpn(*_inputs())
    assert tuple(out[3].shape[2:]) == (3, 5)
    for l, t in enumerate(out):
        want = torch.from_numpy(FIX["%s_out%d" % (case, l)]).double()
        assert t.shape == want.shape, l
        assert float((t - want).abs().max()) <= 1e-5 * float(want.abs().max()), (case, l)
    # the fixture does tell the methods apart: P2..P4 differ from the nearest graph, P5 does not
    for l in range(3):
        want = torch.from_numpy(FIX["%s_out%d" % (case, l)]).double()
        assert float((nearest[l] - want).abs().max()) > 1e-2 * float(want.abs().max()), (case, l)
    assert torch.equal(nearest[3], out[3])
