"""Plain-torch restatement of the reference's optimiser step (lib/nn/optimizer.py:80-104, SGD.step(lr)) and of the
momentum decay of its training loop (upsnet_end2end_train.py:235-240), plus the seeded cases of
tests/golden/reference_sgd.npz.

OracleSGD runs on whichever device its tensors are on: on CPU tensors it is what the fixture pins, on CUDA tensors it is
torch's CUDA ops, which the device kernel must match byte for byte.  The ops are the reference's, one torch op per line:
d = p.grad (+ wd p, in place), buf.mul_(m).add_(d, alpha=group_lr * lr), p.add_(buf, alpha=-1); a buffer is created as
zeros the first time its parameter has a gradient, and a None gradient skips the parameter."""
import hashlib
import json

import numpy as np
import torch


class OracleSGD(torch.optim.Optimizer):
    def __init__(self, params, lr=1, momentum=0, dampening=0, weight_decay=0, nesterov=False):
        assert dampening == 0 and not nesterov
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                                      nesterov=nesterov))

    @torch.no_grad()
    def step(self, lr):
        for group in self.param_groups:
            wd, m = group["weight_decay"], group["momentum"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                d = p.grad
                if wd != 0:
                    d.add_(p, alpha=wd)
                if m != 0:
                    st = self.state[p]
                    if "momentum_buffer" not in st:
                        st["momentum_buffer"] = torch.zeros_like(p)
                    buf = st["momentum_buffer"]
                    buf.mul_(m).add_(d, alpha=group["lr"] * lr)
                    d = buf
                p.add_(d, alpha=-1)


def decay_momentum(optimizer):
    """upsnet_end2end_train.py:238-240: every momentum buffer of optimizer.state_dict() divided by 10 in place."""
    sd = optimizer.state_dict()
    for k in sd["state"].keys():
        if "momentum_buffer" in sd["state"][k]:
            sd["state"][k]["momentum_buffer"].div_(10)


# ---- the fixture cases ------------------------------------------------------------------------
# shapes: the parameters; groups: (group kwargs, indices of the parameters in it); none_until[i]: p.grad of parameter
# i is None before that step; zeros: (parameter, element) pairs set to p = -0.0 and g = -0.0 at every step (the
# signed-zero product of a new buffer); sched: LRSchedule keywords; steps: how many steps from begin_iteration, the
# reference's state_dict is also kept after `mid` of them.
CASES = {
    "groups": dict(seed=1, shapes=[(4, 3), (37,), (1,), (2, 3, 5), (6,)], momentum=0.9, weight_decay=1e-4,
                   groups=[({"lr": 1}, [0, 2]), ({"lr": 2, "weight_decay": 0}, [1, 3]), ({"lr": 1, "weight_decay": 0}, [4])],
                   none_until={3: 2}, zeros=[(4, 0), (4, 5), (2, 0)],
                   sched=dict(lr_schedule="step", base_lr=0.02, max_iteration=9, decay_iteration=[5, 7],
                              warmup_iteration=3), steps=8, mid=6),
    "momentum0": dict(seed=2, shapes=[(5, 7), (3,), (9,)], momentum=0, weight_decay=1e-4,
                      groups=[({"lr": 1}, [0]), ({"lr": 2, "weight_decay": 0}, [1, 2])],
                      none_until={2: 1}, zeros=[(1, 1)],
                      sched=dict(lr_schedule="step", base_lr=0.5, max_iteration=5, decay_iteration=[3],
                                 warmup_iteration=2), steps=5, mid=3),
    "poly_resume": dict(seed=3, shapes=[(11,), (3, 3), (2,)], momentum=0.9, weight_decay=5e-4,
                        groups=[({"lr": 1}, [0, 1]), ({"lr": 2, "weight_decay": 0}, [2])],
                        none_until={0: 3}, zeros=[],
                        sched=dict(lr_schedule="poly", base_lr=0.01, max_iteration=12, decay_iteration=[6],
                                   warmup_iteration=4, begin_iteration=2), steps=8, mid=5),
}


def case_inputs(spec):
    """(initial parameters, grads[step][i] or None), float32 numpy, from the case's seed."""
    params = [np.random.default_rng([spec["seed"], 1000 + i]).standard_normal(s).astype(np.float32)
              for i, s in enumerate(spec["shapes"])]
    grads = []
    for t in range(spec["steps"]):
        gs = []
        for i, s in enumerate(spec["shapes"]):
            if t < spec["none_until"].get(i, 0):
                gs.append(None)
                continue
            g = (np.random.default_rng([spec["seed"], t, i]).standard_normal(s) * 0.1).astype(np.float32)
            gs.append(g)
        grads.append(gs)
    for i, e in spec["zeros"]:
        params[i].reshape(-1)[e] = np.float32(-0.0)
        for gs in grads:
            if gs[i] is not None:
                gs[i].reshape(-1)[e] = np.float32(-0.0)
    return params, grads


def digest(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(b"none" if a is None else np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def inputs_digest(spec):
    params, grads = case_inputs(spec)
    return digest(params + [g for gs in grads for g in gs])


def param_groups(spec, tensors):
    return [dict(kw, params=[tensors[i] for i in idx]) for kw, idx in spec["groups"]]


def decay_momentum_divide(optimizer):
    """decay_momentum with the division the CPU does (float32 b / 10, correctly rounded: b / 10 in float64, then
    rounded), on any device.  torch's CUDA div_(10) multiplies by 1.0f / 10 instead, which can differ by 1 ulp."""
    sd = optimizer.state_dict()
    for k in sd["state"].keys():
        if "momentum_buffer" in sd["state"][k]:
            b = sd["state"][k]["momentum_buffer"]
            b.copy_((b.double() / 10).float())


def run(spec, opt_cls, lr_of, device="cpu", steps=None, start=0, params=None, optimizer=None, decay_fn=decay_momentum):
    """Runs the case's steps [start, steps) with the training loop's order: lr = schedule(it); step(lr); it += 1; decay
    (decay_fn) if it is in decay_iteration.  lr_of(it) -> the learning rate (None: the optimiser has a schedule
    attached, which decays on its own).  -> (parameters, optimiser)."""
    p0, grads = case_inputs(spec)
    if params is None:
        params = [torch.from_numpy(p.copy()).to(device).requires_grad_(True) for p in p0]
    opt = optimizer if optimizer is not None else opt_cls(param_groups(spec, params), lr=1, momentum=spec["momentum"],
                                                          weight_decay=spec["weight_decay"])
    begin = spec["sched"].get("begin_iteration", 0)
    decay = set(spec["sched"]["decay_iteration"])
    for t in range(start, spec["steps"] if steps is None else steps):
        it = begin + t
        for p, g in zip(params, grads[t]):
            p.grad = None if g is None else torch.from_numpy(g.copy()).to(device)
        lr = lr_of(it)
        if lr is None:
            opt.step()
        else:
            opt.step(lr)
        if lr is not None and (it + 1) in decay:
            decay_fn(opt)
    return params, opt


def state_arrays(opt):
    """{parameter index: momentum buffer as numpy} and the group metadata (JSON) of opt.state_dict()."""
    sd = opt.state_dict()
    bufs = {int(k): v["momentum_buffer"].detach().cpu().numpy().copy() for k, v in sd["state"].items()
            if "momentum_buffer" in v}
    meta = json.dumps(sd["param_groups"], sort_keys=True)
    return bufs, meta


def state_dict_from(bufs, meta, device="cpu"):
    """The reference-format state dict of the fixture's arrays."""
    return {"state": {k: {"momentum_buffer": torch.from_numpy(v.copy()).to(device)} for k, v in bufs.items()},
            "param_groups": json.loads(meta)}
