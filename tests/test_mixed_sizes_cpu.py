"""Test-phase image geometry (upsnet_b200.geometry) against the reference's own test-phase path, executed on a list of
original sizes (tests/golden/reference_test_geometry.npz, made by make_reference_test_geometry.py): scale, resized and
padded shape, im_info, the restore size and im_post's size, including which sizes the combined result rejects."""
import os
import types

import numpy as np
import pytest

from upsnet_b200.geometry import image_geometry, prep_scale, scale_for_test_phase

FIX = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_test_geometry.npz"))
CASES = [str(c) for c in FIX["cases"]]


def _config(name):
    dataset, target, max_size = (str(v) for v in FIX["config/" + name])
    return dataset, int(target), int(max_size)


@pytest.mark.parametrize("case", CASES)
def test_geometry_matches_reference(case):
    f = {k.split("/", 1)[1]: FIX[k] for k in FIX.files if k.startswith(case + "/")}
    _, target, max_size = _config(str(f["config"]))
    h, w = (int(v) for v in f["size"])
    g = image_geometry(h, w, target, max_size)
    assert g.scale == float(f["im_scale"])                        # float64, bit for bit
    assert g.resized == tuple(int(v) for v in f["resized"])
    assert g.padded == tuple(int(v) for v in f["padded"])
    assert g.im_info.dtype == np.float32 and np.array_equal(g.im_info.view(np.uint32), f["im_info"][0].view(np.uint32))
    assert g.restored == tuple(int(v) for v in f["restored"])
    assert g.im_post == tuple(int(v) for v in f["im_post"])


def test_fixture_covers_the_edge_cases():
    """The fixture has capped sizes, an h * s on .5, a padded shape shared by two im_info rows, and rejected sizes."""
    rows = {c: {k: FIX[c + "/" + k] for k in ("size", "im_scale", "padded", "im_info", "restored", "im_post", "config")}
            for c in CASES}
    capped = [c for c, r in rows.items() if r["im_scale"] != _config(str(r["config"]))[1] / min(r["size"])]
    assert len(capped) >= 3
    halves = [c for c, r in rows.items() if any(abs(v * float(r["im_scale"]) % 1 - 0.5) < 1e-9 for v in r["size"])]
    assert halves
    shared = {}
    for c, r in rows.items():
        shared.setdefault((str(r["config"]), tuple(r["padded"])), set()).add(tuple(r["im_info"][0].tolist()))
    assert any(len(v) > 1 for v in shared.values())
    rejected = [c for c, r in rows.items() if tuple(r["restored"]) != tuple(r["im_post"])]
    assert sorted(rejected) == ["small_coco_g", "small_coco_h"]


@pytest.mark.parametrize("case", CASES)
def test_combined_rule(case):
    """PipelinedEngine's with_combined check rejects exactly the sizes where the reference's im_post size and restored
    size differ (the merge would fail to broadcast there)."""
    from upsnet_b200.pipeline import PipelinedEngine
    f = {k.split("/", 1)[1]: FIX[k] for k in FIX.files if k.startswith(case + "/")}
    eng = PipelinedEngine(None, target_size=1, max_size=1, max_image_shape=(1, 1), restore_size=True,
                          with_combined=True)
    rejected = tuple(int(v) for v in f["restored"]) != tuple(int(v) for v in f["im_post"])
    if rejected:
        with pytest.raises(ValueError):
            eng._geometry(f["im_info"])
    else:
        g = eng._geometry(f["im_info"])
        assert g["combined_size"] == tuple(int(v) for v in f["im_post"])


def test_prep_scale_is_training_sample_rule():
    """TrainingSample.im_scale is the shared prep_scale."""
    from upsnet_b200.training import TrainingSample
    ts = TrainingSample(scales=(800,), max_size=1333)
    for h, w in [(480, 640), (480, 1000), (1024, 2048), (802, 640)]:
        assert ts.im_scale(800, h, w) == prep_scale(800, 1333, h, w)


def test_scale_for_test_phase():
    net = types.SimpleNamespace(pixel_means=np.zeros(3), rpn_feat_stride=(4, 8, 16, 32, 64))
    cfg = types.SimpleNamespace(network=net, train=types.SimpleNamespace(scales=[800], max_size=1333),
                                test=types.SimpleNamespace(scales=[1024], max_size=2048))
    assert scale_for_test_phase(cfg, "coco") == (800, 1333)          # COCO's test phase reads the train section
    assert scale_for_test_phase(cfg, "cityscapes") == (1024, 2048)
    cfg.test.scales = [800, 1024]
    with pytest.raises(ValueError):
        scale_for_test_phase(cfg, "cityscapes")
    with pytest.raises(ValueError):
        scale_for_test_phase(cfg, "ade20k")


def test_engine_arguments():
    from upsnet_b200.pipeline import PipelinedEngine
    with pytest.raises(ValueError):
        PipelinedEngine(None)                                            # neither im_info nor a size rule
    with pytest.raises(ValueError):
        PipelinedEngine(None, np.array([[64, 64, 1.0]], np.float32), target_size=64, max_size=64, max_image_shape=(8, 8))
