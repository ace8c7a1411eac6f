"""upsnet_b200.SGD / LRSchedule / FlatBucketAllReduce.step on the device: byte-exact against the reference's optimiser
step run with torch's own CUDA ops (tests/sgd_oracle.py), at full UPSNet-50 size, scheduled, under graph replay and
straight from all-reduced bf16 buckets; and against the CPU fixture of the reference's SGD."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist

import sgd_oracle as SO
from upsnet_b200 import _lib
from upsnet_b200.training import SGD, FlatBucketAllReduce, LRSchedule

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FIX = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_sgd.npz"))
PREFIXES = (("resnet_backbone.res3", "resnet_backbone.res4", "resnet_backbone.res5"), ("fpn",), ("rcnn",),
            ("mask_branch",), ("rpn",), ("fcn_head",))


def upsnet50_groups():
    """The shapes of get_params_lr()'s groups for UPSNet-50 (models/resnet_upsnet.py:260-283): conv1, res2 and every
    BatchNorm affine parameter are frozen in the reference (backbone_freeze_at = 2, backbone_fix_bn), so get_params never
    yields them.  -> [(kwargs, [shape, ...])] in the reference's group order (the empty GroupNorm group first)."""
    from upsnet_b200.model import resnet_50_upsnet
    m = resnet_50_upsnet()
    bn = {n + "." + k for n, mod in m.named_modules() if isinstance(mod, torch.nn.BatchNorm2d)
          for k, _ in mod.named_parameters(recurse=False)}
    named = [(n, tuple(p.shape)) for n, p in m.named_parameters() if n not in bn]
    groups = [({"lr": 1, "weight_decay": 0}, [])]
    for pres in PREFIXES:
        for suf, kw in (("weight", {"lr": 1}), ("bias", {"lr": 2, "weight_decay": 0})):
            groups.append((kw, [s for n, s in named if n.startswith(tuple(p + "." for p in pres)) and n.endswith(suf)]))
    return groups


def _make(groups, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [[torch.randn(s, generator=g, device=DEV) * 0.05 for s in shapes] for _, shapes in groups]


def _params(values):
    return [[v.clone().requires_grad_(True) for v in vs] for vs in values]


def _pg(groups, params):
    return [dict(kw, params=ps) for (kw, _), ps in zip(groups, params)]


def _same(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _assert_same_state(pa, oa, pb, ob):
    for x, y in zip(pa, pb):
        assert _same(x.detach(), y.detach())
    sa, sb = oa.state_dict()["state"], ob.state_dict()["state"]
    assert sorted(sa) == sorted(sb)
    for k in sa:
        assert sorted(sa[k]) == sorted(sb[k])
        if "momentum_buffer" in sa[k]:
            assert _same(sa[k]["momentum_buffer"], sb[k]["momentum_buffer"]), k


@pytest.mark.parametrize("momentum", [0.9, 0])
def test_full_upsnet50_parity_with_torch_cuda_ops(momentum):
    groups = upsnet50_groups()
    n = sum(int(np.prod(s)) for _, ss in groups for s in ss)
    assert 40e6 < n < 50e6 and sum(len(ss) for _, ss in groups) == 94
    init = _make(groups, 1)
    pa, pb = _params(init), _params(init)
    flat_a, flat_b = [p for ps in pa for p in ps], [p for ps in pb for p in ps]
    oa = SO.OracleSGD(_pg(groups, pa), lr=1, momentum=momentum, weight_decay=1e-4)
    ob = SGD(_pg(groups, pb), lr=1, momentum=momentum, weight_decay=1e-4)
    none0 = {3, 50, len(flat_a) - 1}                        # no gradient in the first step
    for t, lr in enumerate([0.002, 0.0068, 0.02, 0.02]):
        grads = _make(groups, 100 + t)
        gflat = [g for gs in grads for g in gs]
        for i, (a, b, g) in enumerate(zip(flat_a, flat_b, gflat)):
            a.grad = None if (t == 0 and i in none0) else g.clone()
            b.grad = None if (t == 0 and i in none0) else g.clone()
        oa.step(lr)
        ob.step(lr)
        if t == 1:                                           # a decay iteration, through the training loop's line
            SO.decay_momentum(oa)
            SO.decay_momentum(ob)
        _assert_same_state(flat_a, oa, flat_b, ob)


def _ulps(a, b):
    a, b = np.asarray(a, np.float32).ravel(), np.asarray(b, np.float32).ravel()
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib).max(initial=0)


def _cpu_decay_checked(opt):
    """The reference's decay as the CPU computes it (correct division), after checking that torch's CUDA div_(10), a
    multiply by 1.0f / 10, is within 1 ulp of it on every buffer element."""
    for s in opt.state.values():
        if "momentum_buffer" in s:
            b = s["momentum_buffer"]
            assert _ulps((b.double() / 10).float().cpu().numpy(), b.clone().div_(10).cpu().numpy()) <= 1
    SO.decay_momentum_divide(opt)


@pytest.mark.parametrize("name", sorted(SO.CASES))
def test_device_against_reference_fixture(name):
    """Bit-exact, with the momentum decay done by correct division as the reference's CPU run does it; torch's CUDA
    div_(10) is checked to be within 1 ulp of that at every decay (through the later steps such a difference can grow
    by cancellation, so the run itself decays the CPU's way)."""
    spec = SO.CASES[name]
    sched = LRSchedule(**spec["sched"])
    params, opt = SO.run(spec, SGD, sched, device=DEV, steps=spec["mid"], decay_fn=_cpu_decay_checked)
    for tag in ("mid", "final"):
        if tag == "final":
            params, opt = SO.run(spec, SGD, sched, device=DEV, start=spec["mid"], params=params, optimizer=opt,
                                 decay_fn=_cpu_decay_checked)
        bufs, meta = SO.state_arrays(opt)
        p = "case/%s/%s/" % (name, tag)
        assert meta == str(FIX[p + "meta"])
        got = [t.detach().cpu().numpy() for t in params] + [bufs[k] for k in sorted(bufs)]
        want = [FIX[p + "param%d" % i] for i in range(len(params))] + [FIX[p + "buf%d" % k] for k in sorted(bufs)]
        assert sorted(bufs) == sorted(int(k.rsplit("buf", 1)[1]) for k in FIX.files if k.startswith(p + "buf"))
        for g_, w_ in zip(got, want):
            assert np.array_equal(g_.view(np.uint32), w_.view(np.uint32)), (tag, _ulps(g_, w_))


def _case_pair(name):
    spec = SO.CASES[name]
    return spec, LRSchedule(**spec["sched"])


@pytest.mark.parametrize("name", ["groups", "poly_resume"])
def test_scheduled_step_matches_step_lr_and_loop_decay(name):
    spec, sched = _case_pair(name)
    pa, oa = SO.run(spec, SGD, sched, device=DEV)                       # step(schedule(i)) + state_dict decay
    p0, _ = SO.case_inputs(spec)
    pb = [torch.from_numpy(p.copy()).to(DEV).requires_grad_(True) for p in p0]
    ob = SGD(SO.param_groups(spec, pb), lr=1, momentum=spec["momentum"], weight_decay=spec["weight_decay"])
    ob.attach_schedule(sched)
    pb, ob = SO.run(spec, SGD, lambda it: None, device=DEV, params=pb, optimizer=ob)
    _assert_same_state(pa, oa, pb, ob)
    assert ob.iteration == sched.begin_iteration + spec["steps"]
    with pytest.raises(_lib.UpsnetError):
        ob.step(0.1)
    with pytest.raises(_lib.UpsnetError):
        oa.step()


def test_graph_replay_equals_eager_steps():
    groups = [({"lr": 1}, [(64, 3, 3, 3), (1024, 129), (37,)]), ({"lr": 2, "weight_decay": 0}, [(1,), (36,), (4099,)])]
    sched = LRSchedule(base_lr=0.02, max_iteration=40, decay_iteration=[6], warmup_iteration=4)
    init = _make(groups, 5)
    runs = []
    for use_graph in (False, True):
        ps = _params(init)
        opt = SGD(_pg(groups, ps), lr=1, momentum=0.9, weight_decay=1e-4)
        opt.attach_schedule(sched)
        flat = [p for g in ps for p in g]
        for p in flat:
            p.grad = torch.zeros_like(p)
        gvals = [[g for gs in _make(groups, 200 + t) for g in gs] for t in range(9)]
        for p, g in zip(flat, gvals[0]):
            p.grad.copy_(g)
        opt.step()                                                      # eager: uploads the chunk table
        graph = None
        if use_graph:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                opt.step()
        for t in range(1, 9):
            for p, g in zip(flat, gvals[t]):
                p.grad.copy_(g)
            graph.replay() if use_graph else opt.step()
        torch.cuda.synchronize()
        runs.append((flat, opt))
    (fa, oa), (fb, ob) = runs
    _assert_same_state(fa, oa, fb, ob)
    assert oa.iteration == ob.iteration == 9


def _nccl_group(tmp_path):
    store = dist.FileStore(str(tmp_path / "store"), 1)
    dist.init_process_group("nccl", store=store, rank=0, world_size=1, device_id=DEV)


def _bucket_case():
    # odd sizes so that bucket segments start at odd bf16 offsets; 1 and 37 elements; a large tensor that spans chunks
    return [({"lr": 1}, [(37,), (1,), (300, 301), (9,), (64, 3, 3, 3)]), ({"lr": 2, "weight_decay": 0}, [(36,), (1,), (5,)])]


def test_fused_bucket_step_equals_start_finish_step(tmp_path):
    torch.cuda.set_device(DEV)
    _nccl_group(tmp_path)
    try:
        groups = _bucket_case()
        init = _make(groups, 7)
        pa, pb = _params(init), _params(init)
        fa, fb = [p for g in pa for p in g], [p for g in pb for p in g]
        oa = SGD(_pg(groups, pa), lr=1, momentum=0.9, weight_decay=1e-4)
        ob = SGD(_pg(groups, pb), lr=1, momentum=0.9, weight_decay=1e-4)
        ara = FlatBucketAllReduce(fa, bucket_bytes=60000)
        arb = FlatBucketAllReduce(fb, bucket_bytes=60000)
        assert len(arb.buckets) >= 2
        for t, lr in enumerate([0.01, 0.02, 0.02]):
            gs = [g for gg in _make(groups, 300 + t) for g in gg]
            for i, (a, b, g) in enumerate(zip(fa, fb, gs)):
                a.grad = None if (t == 0 and i == 1) else g.clone()
                b.grad = None if (t == 0 and i == 1) else g.clone()
            ara.start().finish()
            oa.step(lr)
            arb.step(ob, lr)
            if t == 0:
                assert fb[1].grad is None                               # the fused path does not write p.grad
            for a, b in zip(fa, fb):
                assert _same(a.detach(), b.detach())
            for a, b in zip(fa, fb):
                assert _same(oa.state[a]["momentum_buffer"], ob.state[b]["momentum_buffer"])
        with pytest.raises(_lib.UpsnetError):
            FlatBucketAllReduce(fb[:-1]).step(ob, 0.1)
    finally:
        dist.destroy_process_group()


def test_apply_from_bucket_at_world_3_matches_division():
    groups = _bucket_case()
    init = _make(groups, 9)
    pa, pb = _params(init), _params(init)
    fa, fb = [p for g in pa for p in g], [p for g in pb for p in g]
    oa = SO.OracleSGD(_pg(groups, pa), lr=1, momentum=0.9, weight_decay=1e-4)
    ob = SGD(_pg(groups, pb), lr=1, momentum=0.9, weight_decay=1e-4)
    n = sum(p.numel() for p in fb)
    for t in range(2):
        flat = (torch.randn(n, device=DEV, generator=torch.Generator(device=DEV).manual_seed(t)) * 3).bfloat16()
        off = 0
        for p in fa:
            p.grad = (flat[off:off + p.numel()].to(torch.float32) / 3).view_as(p)
            off += p.numel()
        oa.step(0.02)
        table, cnt = ob._bucket_table(fb, flat, 3)
        ob._apply(table, cnt, 0.02)
        _assert_same_state(fa, oa, fb, ob)


def _two_rank_worker(rank, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=dev)
    try:
        groups = _bucket_case()
        g = torch.Generator(device=dev).manual_seed(11)
        init = [[torch.randn(s, generator=g, device=dev) for s in ss] for _, ss in groups]
        ps = [[[v.clone().requires_grad_(True) for v in vs] for vs in init] for _ in range(2)]
        flats = [[p for gg in x for p in gg] for x in ps]
        opts = [SGD(_pg(groups, x), lr=1, momentum=0.9, weight_decay=1e-4) for x in ps]
        ars = [FlatBucketAllReduce(f, bucket_bytes=60000) for f in flats]
        for t in range(2):
            gr = torch.Generator(device=dev).manual_seed(100 * rank + t)
            gs = [torch.randn(p.shape, generator=gr, device=dev) for p in flats[0]]
            for f in flats:
                for p, gg in zip(f, gs):
                    p.grad = gg.clone()
            ars[0].start().finish()
            opts[0].step(0.02)
            ars[1].step(opts[1], 0.02)
        ok = all(_same(a.detach(), b.detach()) for a, b in zip(*flats))
        q.put((rank, ok))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_fused_bucket_step_two_ranks():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_rank_worker, args=(r, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=300) for _ in procs]
    finally:
        for p in procs:
            p.join(120)
    assert all(ok for _, ok in res), res


def test_misaligned_parameters_and_state_aliases():
    base = torch.randn(200, device=DEV)
    groups = [({"lr": 1}, None), ({"lr": 2, "weight_decay": 0}, None)]
    def views():
        b = base.clone()
        return [[torch.nn.Parameter(b[1:38]), torch.nn.Parameter(b[38:39])], [torch.nn.Parameter(b[41:150])]]
    pa, pb = views(), views()
    assert pb[0][0].data_ptr() % 16 == 4
    oa = SO.OracleSGD(_pg(groups, pa), lr=1, momentum=0.9, weight_decay=1e-4)
    ob = SGD(_pg(groups, pb), lr=1, momentum=0.9, weight_decay=1e-4)
    fa, fb = [p for g in pa for p in g], [p for g in pb for p in g]
    for t in range(3):
        for a, b in zip(fa, fb):
            g = torch.randn(a.shape, device=DEV)
            a.grad, b.grad = g.clone(), g.clone()
        oa.step(0.05)
        ob.step(0.05)
        SO.decay_momentum(oa)
        SO.decay_momentum(ob)
    _assert_same_state(fa, oa, fb, ob)
    sd = ob.state_dict()["state"]
    for k, p in enumerate(fb):
        buf = sd[k]["momentum_buffer"]
        assert buf.data_ptr() == ob.state[p]["momentum_buffer"].data_ptr() and buf.data_ptr() % 16 == 0
        assert ob._flat.data_ptr() <= buf.data_ptr() < ob._flat.data_ptr() + 4 * ob._flat.numel()


@pytest.mark.parametrize("name", ["groups", "poly_resume"])
def test_load_reference_state_then_step(name):
    spec, sched = _case_pair(name)
    p = "case/%s/mid/" % name
    bufs = {int(k.rsplit("buf", 1)[1]): FIX[k] for k in FIX.files if k.startswith(p + "buf")}
    runs = []
    for cls in (SO.OracleSGD, SGD):
        params = [torch.from_numpy(FIX[p + "param%d" % i].copy()).to(DEV).requires_grad_(True)
                  for i in range(len(spec["shapes"]))]
        opt = cls(SO.param_groups(spec, params), lr=1, momentum=spec["momentum"], weight_decay=spec["weight_decay"])
        opt.load_state_dict(SO.state_dict_from(bufs, str(FIX[p + "meta"]), DEV))
        if cls is SGD:
            views = {id(v) for v in opt._views.values()}
            assert all(id(s["momentum_buffer"]) in views for s in opt.state.values() if "momentum_buffer" in s)
        runs.append(SO.run(spec, cls, sched, device=DEV, start=spec["mid"], params=params, optimizer=opt,
                           decay_fn=SO.decay_momentum_divide))
    _assert_same_state(runs[0][0], runs[0][1], runs[1][0], runs[1][1])
    q = "case/%s/final/" % name
    bufs, _ = SO.state_arrays(runs[1][1])
    for i, t in enumerate(runs[1][0]):
        assert np.array_equal(t.detach().cpu().numpy().view(np.uint32), FIX[q + "param%d" % i].view(np.uint32))
    for k, v in bufs.items():
        assert np.array_equal(v.view(np.uint32), FIX[q + "buf%d" % k].view(np.uint32))


def test_errors(tmp_path):
    E = _lib.UpsnetError
    p = torch.nn.Parameter(torch.zeros(5, device=DEV))
    with pytest.raises(E):
        SGD([torch.nn.Parameter(torch.zeros(5))], lr=1)
    with pytest.raises(E):
        SGD([torch.nn.Parameter(torch.zeros(5, device=DEV, dtype=torch.float64))], lr=1)
    with pytest.raises(E):
        SGD([p, torch.nn.Parameter(torch.zeros(5))], lr=1)
    with pytest.raises(E):
        SGD([p], lr=1, momentum=0.9, nesterov=True)
    with pytest.raises(E):
        SGD([p], lr=1, momentum=0.9, dampening=0.5)
    with pytest.raises(E):
        LRSchedule(lr_schedule="exp", base_lr=0.1, max_iteration=10)
    opt = SGD([p], lr=1, momentum=0.9)
    p.grad = torch.ones_like(p)
    with pytest.raises(E):
        opt.step()
    opt.attach_schedule(LRSchedule(base_lr=0.1, max_iteration=10))
    with pytest.raises(E):
        opt.step(0.1)
    q = torch.nn.Parameter(torch.zeros(5, device=DEV))
    _nccl_group(tmp_path)
    try:
        with pytest.raises(E):
            FlatBucketAllReduce([p, q]).step(opt)
    finally:
        dist.destroy_process_group()
