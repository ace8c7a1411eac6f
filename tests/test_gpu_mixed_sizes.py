"""Images of different sizes through the static engine: one captured graph per padded input shape and lane, with the
image geometry (im_info) a device input of the graph, and the mixed-size PipelinedEngine.

Cityscapes configuration: the fused maskroi_prepare kernel; COCO configuration: R*(C-1) = 1000*80 is above the fused
kernel's limit, so StaticMaskROI's torch path clips against the device row.  Reduced depth and small sizes."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_sample_cases as TS  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FIX = np.load(os.path.join(HERE, "golden", "reference_test_geometry.npz"))
# target 96, max_size 160: the fixture's coco_small configuration
SMALL = (96, 160)
# (A, B share a padded shape with different im_info; C has another padded shape)
SEQ = {"cityscapes": [(100, 150), (100, 140), (50, 60)],       # 128x192, 128x192, 128x160 at 128 / 256
       "coco": [(64, 90), (64, 100), (60, 200)]}               # 96x160, 96x160, 64x160 at 96 / 160
SIZES = {"cityscapes": (128, 256), "coco": SMALL}


def _model(name):
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    cfg = UPSNetConfig.cityscapes_r50() if name == "cityscapes" else UPSNetConfig.coco_r50()
    return synthetic_model(cfg, depth=(1, 1, 1, 1), seed=3, device=DEV)


def _raw(h, w, seed):
    return torch.from_numpy(TS.image_bgr(h, w, seed)).pin_memory()


def _inputs(sizes, rule, seed0=70):
    from upsnet_b200 import operators as ops
    from upsnet_b200.geometry import image_geometry
    out = []
    for i, (h, w) in enumerate(sizes):
        g = image_geometry(h, w, *rule)
        blob, _ = ops.prep_image(_raw(h, w, seed0 + i).to(DEV), TS.PIXEL_MEANS, g.scale)
        out.append((blob, g.im_info[None]))
    return out


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("name", ["cityscapes", "coco"])
def test_interleaved_replay(name):
    """A, B, C, A, B through model.forward with graphs == the eager static forward of each image; two graphs per lane."""
    import upsnet_b200 as U
    m = _model(name)
    imgs = _inputs(SEQ[name], SIZES[name])
    (xa, ia), (xb, ib), (xc, ic) = imgs
    assert xa.shape == xb.shape != xc.shape and not np.array_equal(ia, ib)
    U.set_precision("bf16x3")
    try:
        with torch.no_grad():
            m.use_cuda_graph = False
            want = [{k: v.clone() for k, v in m({"data": x, "im_info": i}).items() if torch.is_tensor(v)} for x, i in imgs]
            # the case discriminates: B under A's im_info is clipped differently
            m.keep_intermediates = True
            own = m({"data": xb, "im_info": ib})["_intermediates"]
            other = m({"data": xb, "im_info": ia})["_intermediates"]
            m.keep_intermediates = False
            assert not torch.equal(own["rois"], other["rois"])
            m.use_cuda_graph = True
            m._graphs = {}
            for j in (0, 1, 2, 0, 1):
                x, i = imgs[j]
                got = {k: v for k, v in m({"data": x, "im_info": i}).items() if torch.is_tensor(v)}
                _same(got, want[j])
            assert len(m._graphs) == 2 and all(k[-1] == 0 for k in m._graphs)
    finally:
        U.set_precision("fp32")
        m.use_cuda_graph, m.keep_intermediates = True, False


def test_lane_pool_is_shared():
    """All graphs of a lane share one memory pool: a second, smaller shape adds less than the first capture did."""
    import upsnet_b200 as U
    m = _model("cityscapes")
    big, small = _inputs([(128, 256)], (256, 512))[0], _inputs([(64, 128)], (128, 256))[0]
    U.set_precision("bf16x3")
    try:
        with torch.no_grad():
            m({"data": small[0][..., :64, :64].contiguous(), "im_info": np.array([[64, 64, 1.0]], np.float32)})
            m._graphs, m._pools = {}, {}
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            r0 = torch.cuda.memory_reserved()
            m._run_static(big[0], big[1][0])
            torch.cuda.synchronize()
            r1 = torch.cuda.memory_reserved()
            m._run_static(small[0], small[1][0])
            torch.cuda.synchronize()
            r2 = torch.cuda.memory_reserved()
    finally:
        U.set_precision("fp32")
    assert big[0].shape[-2:] == (256, 512) and small[0].shape[-2:] == (128, 256)
    assert len(m._graphs) == 2 and len(m._pools) == 1
    assert r2 - r1 < r1 - r0, (r0, r1, r2)


def test_pipeline_mixed_sizes_parity():
    """Mixed-size PipelinedEngine (depth 2, lanes 2, masks, unified, restore, combined) == a fixed-size engine built for
    each image's im_info and run on that image alone.  Slot 0 sees 96x160 then 96x96, slot 1 128x96 then 64x160; an
    image whose im_post size differs from its restored size raises at submit and leaves the engine usable."""
    import upsnet_b200 as U
    m = _model("cityscapes")
    from upsnet_b200.geometry import image_geometry
    sizes = [(64, 90), (81, 64), (70, 70), (60, 200), (115, 112), (64, 100), (65, 80)]
    raws = [_raw(h, w, 90 + i) for i, (h, w) in enumerate(sizes)]
    kw = dict(with_masks=True, with_unified=True, restore_size=True, with_combined=True, combined_score_threshold=0.05,
              stuff_area_limit=256)
    U.set_precision("bf16x3")
    try:
        eng = U.PipelinedEngine(m, depth=2, lanes=2, target_size=SMALL[0], max_size=SMALL[1], max_image_shape=(120, 200),
                                **kw)
        got, pending, rejected = {}, [], []
        for i, r in enumerate(raws):
            try:
                pending.append((i, eng.submit(r)))
            except ValueError:
                rejected.append(i)
                continue
            if len(pending) == 2:
                j, t = pending.pop(0)
                got[j] = {k: v.clone() for k, v in eng.result(t).items()}
        for j, t in pending:
            got[j] = {k: v.clone() for k, v in eng.result(t).items()}
        assert rejected == [4]
        shapes = {image_geometry(h, w, *SMALL).padded for h, w in sizes}
        assert len(shapes) >= 4
        instances = 0
        for i, r in enumerate(raws):
            if i in rejected:
                continue
            g = image_geometry(*sizes[i], *SMALL)
            ref = U.PipelinedEngine(m, g.im_info[None], depth=2, im_scale=g.scale, **kw)
            want = ref.result(ref.submit(r))
            _same(got[i], want)
            assert got[i]["fcn_outputs"].shape == (1,) + sizes[i]
            assert np.array_equal(got[i]["im_info"].numpy()[0], g.im_info)
            instances += int((got[i]["pan_2ch_combined"][..., 1] > 0).sum())
        assert instances > 0
    finally:
        U.set_precision("fp32")


def test_staged_blobs_match_fixture():
    """The blob the mixed-size engine stages for each of the fixture's small cases == the reference's padded blob, zero
    padding included; one slot, so the 64x160 blob is staged where a 128x96 one was."""
    import upsnet_b200 as U
    m = _model("coco")
    names = ["small_coco_e", "small_coco_d", "small_coco_b"]           # 128x96, 64x160, 96x160
    U.set_precision("bf16")
    try:
        eng = U.PipelinedEngine(m, depth=1, target_size=SMALL[0], max_size=SMALL[1], max_image_shape=(120, 200))
        for n in names:
            h, w = (int(v) for v in FIX[n + "/size"])
            want = FIX[n + "/blob"]
            eng.result(eng.submit(_raw(h, w, int(FIX[n + "/image_seed"]))))
            Hp, Wp = want.shape[2:]
            got = eng._slots[0]["x"][:3 * Hp * Wp].view(1, 3, Hp, Wp).cpu().numpy()
            ho, wo = (int(v) for v in FIX[n + "/resized"])
            assert not got[:, :, ho:].any() and not got[:, :, :, wo:].any()
            assert np.abs(got - want).max() < 1e-3 * max(1.0, np.abs(want).max() / 30), n
    finally:
        U.set_precision("fp32")
