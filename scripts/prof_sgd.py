"""The optimiser step on the UPSNet-50 parameter set (get_params_lr()'s groups, tests/test_gpu_sgd.upsnet50_groups):
python scripts/prof_sgd.py [steps]

Reported per step, as CUDA events over `steps` steps per round after a warm-up, rounds alternated:
  * oracle:        the reference's SGD.step(lr) restated in plain torch (tests/sgd_oracle.py), issued from Python;
  * step_lr:       upsnet_b200.SGD.step(lr) (the chunk-table key check on the host, one apply launch);
  * graph_sched:   the scheduled step (apply + advance) captured once in a CUDA graph and replayed;
  * bucket_unfused / bucket_fused: start(); finish(); step(lr) against FlatBucketAllReduce.step(opt, lr) on a one-rank
                   NCCL group (25 MB bf16 buckets);
  * torch_foreach / torch_fused: torch.optim.SGD(foreach=True) and (fused=True), for context only (their update rule
                   differs from the reference's).
The apply kernel alone is timed as graph replays of 20 launches, from float32 gradients (20 bytes per parameter: p and
the buffer read and written, the gradient read) and from a bf16 bucket (18 bytes); achieved GB/s is those bytes over the
kernel time, against the 3.35 TB/s of the H100 SXM data sheet.  The card and its power limit are read in the same run.
There is no fallback: without a GPU the script fails."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import sgd_oracle as SO  # noqa: E402
from prof_rpn_targets import card, events_ms  # noqa: E402
from test_gpu_sgd import upsnet50_groups  # noqa: E402
from upsnet_b200.training import SGD, FlatBucketAllReduce, LRSchedule  # noqa: E402

DEV = torch.device("cuda", 0)
ROUNDS = 3
HBM = 3.35e12


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    torch.cuda.set_device(DEV)
    groups = upsnet50_groups()
    g = torch.Generator(device=DEV).manual_seed(0)
    params = [[(torch.randn(s, generator=g, device=DEV) * 0.05).requires_grad_(True) for s in ss] for _, ss in groups]
    flat = [p for ps in params for p in ps]
    for p in flat:
        p.grad = torch.randn(p.shape, generator=g, device=DEV) * 1e-3
    n = sum(p.numel() for p in flat)
    pg = lambda: [dict(kw, params=ps) for (kw, _), ps in zip(groups, params)]  # noqa: E731
    kw = dict(lr=1, momentum=0.9, weight_decay=1e-4)

    oracle = SO.OracleSGD(pg(), **kw)
    ours = SGD(pg(), **kw)
    sched = SGD(pg(), **kw)
    sched.attach_schedule(LRSchedule(base_lr=0.02, max_iteration=10 ** 6, decay_iteration=[5 * 10 ** 5],
                                     warmup_iteration=1500))
    fe = torch.optim.SGD(pg(), momentum=0.9, weight_decay=1e-4, foreach=True)
    fu = torch.optim.SGD(pg(), momentum=0.9, weight_decay=1e-4, fused=True)
    sched.step()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sched.step()

    # the apply kernel alone: 20 launches per replay, float32 gradients and a bf16 bucket (world 1)
    table, cnt = ours._grad_table()
    bucket = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    btable, bcnt = ours._bucket_table(flat, bucket, 1)
    kgraphs = {}
    for name, (tb, c) in (("apply_f32", (table, cnt)), ("apply_bf16", (btable, bcnt))):
        ours._apply(tb, c, 0.02)
        kg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(kg):
            for _ in range(20):
                ours._apply(tb, c, 0.02)
        kgraphs[name] = kg

    store_dir = tempfile.mkdtemp()
    dist.init_process_group("nccl", store=dist.FileStore(os.path.join(store_dir, "store"), 1), rank=0, world_size=1,
                            device_id=DEV)
    try:
        ar_u = FlatBucketAllReduce(flat)
        ar_f = FlatBucketAllReduce(flat)
        bo_u, bo_f = SGD(pg(), **kw), SGD(pg(), **kw)

        def bucket_unfused(i=0):
            ar_u.start().finish()
            bo_u.step(0.02)

        cases = {
            "oracle": lambda i=0: oracle.step(0.02),
            "step_lr": lambda i=0: ours.step(0.02),
            "graph_sched": lambda i=0: graph.replay(),
            "bucket_unfused": bucket_unfused,
            "bucket_fused": lambda i=0: ar_f.step(bo_f, 0.02),
            "torch_foreach": lambda i=0: fe.step(),
            "torch_fused": lambda i=0: fu.step(),
        }
        for fn in cases.values():
            for _ in range(3):
                fn()
        for kg in kgraphs.values():
            kg.replay()
        torch.cuda.synchronize()
        times = {k: [] for k in list(cases) + list(kgraphs)}
        for _ in range(ROUNDS):
            for k, fn in cases.items():
                times[k].append(events_ms(fn, steps))
            for k, kg in kgraphs.items():
                times[k].append(events_ms(lambda i=0: kg.replay(), max(steps // 5, 4)) / 20)
    finally:
        dist.destroy_process_group()
    best = {k: min(v) for k, v in times.items()}
    bw = {"apply_f32": 20 * n, "apply_bf16": 18 * n}
    out = {"card": card(), "params": n, "tensors": len(flat), "steps_per_round": steps, "rounds": ROUNDS,
           "ms_per_step_min": {k: round(v, 4) for k, v in best.items()},
           "ms_per_step_all": {k: [round(x, 4) for x in v] for k, v in times.items()},
           "apply_GBps": {k: round(b / (best[k] * 1e-3) / 1e9, 1) for k, b in bw.items()},
           "apply_share_of_3.35TBps": {k: round(b / (best[k] * 1e-3) / HBM, 3) for k, b in bw.items()}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
