"""The optimiser's oracle and learning-rate schedule against tests/golden/reference_sgd.npz (the reference's SGD,
adjust_learning_rate and shipped yaml schedules, executed): bit-exact on CPU."""
import ast
import hashlib
import os

import numpy as np
import pytest
import torch

import sgd_oracle as SO
from upsnet_b200 import _lib
from upsnet_b200.training import SGD, LRSchedule

FIX = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_sgd.npz"))


def _schedule(spec):
    return LRSchedule(**spec["sched"])


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("name", sorted(SO.CASES))
def test_oracle_matches_reference_sgd(name):
    spec = SO.CASES[name]
    p = "case/%s/" % name
    assert str(FIX[p + "inputs_sha256"]) == SO.inputs_digest(spec)
    sched = _schedule(spec)
    begin = spec["sched"].get("begin_iteration", 0)
    assert np.array_equal(FIX[p + "lr"], [sched(begin + t) for t in range(spec["steps"])])
    params, opt = SO.run(spec, SO.OracleSGD, sched, steps=spec["mid"])
    for tag in ("mid", "final"):
        if tag == "final":
            params, opt = SO.run(spec, SO.OracleSGD, sched, start=spec["mid"], params=params, optimizer=opt)
        bufs, meta = SO.state_arrays(opt)
        assert meta == str(FIX[p + tag + "/meta"])
        for i, t in enumerate(params):
            assert np.array_equal(_bits(t.detach().numpy()), _bits(FIX[p + tag + "/param%d" % i])), (tag, i)
        want = sorted(int(k.rsplit("buf", 1)[1]) for k in FIX.files if k.startswith(p + tag + "/buf"))
        assert sorted(bufs) == want
        for k, v in bufs.items():
            assert np.array_equal(_bits(v), _bits(FIX[p + tag + "/buf%d" % k])), (tag, k)


def test_fixture_pins_the_reference_behaviours():
    # None gradients create no buffer (parameter 3 of 'groups' has one only from step 2 on; 'momentum0' has none at
    # all), and the signed-zero case keeps -0.0 where a buffer starting at -0 would give +0
    assert "case/groups/mid/buf3" in FIX.files and not any(k.startswith("case/momentum0/final/buf") for k in FIX.files)
    p4 = FIX["case/groups/final/param4"]
    assert np.signbit(p4[0]) and p4[0] == 0 and np.signbit(p4[5])
    assert not np.signbit(FIX["case/groups/final/buf4"][0])


def _train(key):
    return dict(ast.literal_eval(str(FIX[key])))


LR_KEYS = sorted({k.rsplit("/", 1)[0] for k in FIX.files if k.startswith("lr/")})


@pytest.mark.parametrize("key", LR_KEYS)
def test_lr_schedule_matches_reference(key):
    tr = _train(key + "/train")
    s = LRSchedule(lr_schedule=tr["lr_schedule"], base_lr=tr["lr"], max_iteration=tr["max_iteration"],
                   decay_iteration=tr["decay_iteration"], warmup_iteration=tr["warmup_iteration"],
                   begin_iteration=tr["begin_iteration"])
    its = FIX[key + "/iters"]
    assert [s(int(i)) for i in its] == FIX[key + "/values"].tolist()
    table = s.table()
    assert hashlib.sha256(table.tobytes()).hexdigest() == str(FIX[key + "/sha256"])
    flags = s.decay_flags()
    assert flags.sum() == sum(1 for d in tr["decay_iteration"] if tr["begin_iteration"] < d <= tr["max_iteration"])


def test_lr_schedule_from_config_and_errors():
    import types
    tr = types.SimpleNamespace(lr_schedule="step", lr=0.02, max_iteration=100, decay_iteration=[50, 80],
                               warmup_iteration=10, begin_iteration=20)
    s = LRSchedule(types.SimpleNamespace(train=tr))
    assert s.table().shape == (80,) and s(60) == 0.02 * 0.1 ** 1
    assert np.flatnonzero(s.decay_flags()).tolist() == [49 - 20, 79 - 20]
    with pytest.raises(_lib.UpsnetError):
        LRSchedule(lr_schedule="cosine", base_lr=0.1, max_iteration=10)
    with pytest.raises(_lib.UpsnetError):
        LRSchedule(base_lr=0.1, max_iteration=10, begin_iteration=10)


@pytest.mark.parametrize("name", sorted(SO.CASES))
def test_state_dict_round_trip_in_reference_format(name):
    spec = SO.CASES[name]
    p = "case/%s/mid/" % name
    bufs = {int(k.rsplit("buf", 1)[1]): FIX[k] for k in FIX.files if k.startswith(p + "buf")}
    params = [torch.zeros(s, requires_grad=True) for s in spec["shapes"]]
    opt = SO.OracleSGD(SO.param_groups(spec, params), lr=1, momentum=spec["momentum"],
                       weight_decay=spec["weight_decay"])
    opt.load_state_dict(SO.state_dict_from(bufs, str(FIX[p + "meta"])))
    got, meta = SO.state_arrays(opt)
    assert meta == str(FIX[p + "meta"]) and sorted(got) == sorted(bufs)
    for k in bufs:
        assert np.array_equal(_bits(got[k]), _bits(bufs[k]))
    keys = {k for g in opt.state_dict()["param_groups"] for k in g}
    assert keys == {"lr", "momentum", "dampening", "weight_decay", "nesterov", "params"}


def test_sgd_rejects_what_it_does_not_build():
    p = torch.nn.Parameter(torch.zeros(3))
    with pytest.raises(_lib.UpsnetError):          # CPU parameters
        SGD([p], lr=1)
    with pytest.raises(_lib.UpsnetError):
        SGD([p], lr=1, momentum=0.9, nesterov=True)
    with pytest.raises(_lib.UpsnetError):
        SGD([p], lr=1, momentum=0.9, dampening=0.1)
