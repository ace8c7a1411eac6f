"""Generates tests/golden/reference_sgd.npz by EXECUTING the reference's optimiser and learning-rate schedule (build
container only: /root/reference is not present on the GPU box).  Run: python tests/golden/make_reference_sgd.py

* lib/nn/optimizer.py's SGD is imported unmodified, with lib.utils.logging stubbed (its logger is only printed to).
* lr_poly, get_step_index, lr_factor and adjust_learning_rate are taken from upsnet_end2end_train.py by their AST (the
  script itself cannot be imported: it parses arguments and pulls in the whole training stack at import time).
* The train: sections of the seven shipped experiments/*.yaml, over config.py's defaults (lr_schedule 'step',
  begin_iteration 0).

Written: for each case of tests/sgd_oracle.CASES, run on CPU float32 tensors with the training loop's order (lr of the
iteration, step(lr), iteration + 1, the state_dict decay loop), the sha256 of the seeded inputs, the learning rates, and
the parameters and the optimiser's state_dict (buffers + group metadata) after `mid` steps and after all of them.  For
each yaml and each schedule ('step' as shipped, and 'poly'), the sha256 of the float64 learning-rate table over
[begin_iteration, max_iteration) and its values at and around every warm-up and decay boundary.  The archive is written
with fixed member timestamps, so a second run gives the same bytes."""
import ast
import glob
import hashlib
import importlib.util
import io
import os
import sys
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import sgd_oracle as SO  # noqa: E402

REF = "/root/reference"
LR_FUNCS = ("lr_poly", "get_step_index", "lr_factor", "adjust_learning_rate")


def reference_sgd():
    logging = types.ModuleType("lib.utils.logging")
    logging.logger = None
    for name in ("lib", "lib.utils"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["lib.utils.logging"] = logging
    spec = importlib.util.spec_from_file_location("ref_optimizer", os.path.join(REF, "lib", "nn", "optimizer.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.SGD


def reference_lr():
    path = os.path.join(REF, "upsnet", "upsnet_end2end_train.py")
    tree = ast.parse(open(path).read(), path)
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in LR_FUNCS]
    assert sorted(n.name for n in body) == sorted(LR_FUNCS)
    ns = {}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns["adjust_learning_rate"]


def yaml_trains():
    import yaml
    out = {}
    for f in sorted(glob.glob(os.path.join(REF, "upsnet", "experiments", "*.yaml"))):
        tr = dict(lr_schedule="step", begin_iteration=0)            # upsnet/config/config.py defaults
        tr.update(yaml.safe_load(open(f))["train"])
        out[os.path.splitext(os.path.basename(f))[0]] = tr
    return out


def _config(tr):
    return types.SimpleNamespace(train=types.SimpleNamespace(**tr))


def boundaries(tr):
    b, m = tr["begin_iteration"], tr["max_iteration"]
    its = {b, b + 1, m - 1}
    for x in [tr["warmup_iteration"]] + list(tr["decay_iteration"]):
        its.update((x - 1, x, x + 1))
    return np.array(sorted(i for i in its if b <= i < m), np.int64)


def save_npz(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    import torch
    SGD = reference_sgd()
    adjust = reference_lr()
    out = {}
    for name, spec in SO.CASES.items():
        cfg = _config(dict(spec["sched"], lr=spec["sched"]["base_lr"]))
        lr_of = lambda it: adjust(None, it, cfg)  # noqa: E731
        p = "case/%s/" % name
        begin = spec["sched"].get("begin_iteration", 0)
        out[p + "inputs_sha256"] = np.str_(SO.inputs_digest(spec))
        out[p + "lr"] = np.array([lr_of(begin + t) for t in range(spec["steps"])], np.float64)
        params, opt = SO.run(spec, SGD, lr_of, steps=spec["mid"])
        for tag in ("mid", "final"):
            if tag == "final":
                params, opt = SO.run(spec, SGD, lr_of, start=spec["mid"], params=params, optimizer=opt)
            bufs, meta = SO.state_arrays(opt)
            out[p + tag + "/meta"] = np.str_(meta)
            for i, t in enumerate(params):
                out[p + tag + "/param%d" % i] = t.detach().numpy().copy()
            for k, v in bufs.items():
                out[p + tag + "/buf%d" % k] = v
        print("case", name, "steps", spec["steps"], "buffers", sorted(bufs))
    for yname, tr in yaml_trains().items():
        for sched in ("step", "poly"):
            t = dict(tr, lr_schedule=sched)
            cfg = _config(t)
            table = np.array([adjust(None, i, cfg) for i in range(t["begin_iteration"], t["max_iteration"])], np.float64)
            its = boundaries(t)
            p = "lr/%s/%s/" % (yname, sched)
            out[p + "sha256"] = np.str_(hashlib.sha256(table.tobytes()).hexdigest())
            out[p + "iters"] = its
            out[p + "values"] = table[its - t["begin_iteration"]]
            out[p + "train"] = np.str_(repr(sorted((k, t[k]) for k in ("lr_schedule", "lr", "max_iteration",
                                                                        "decay_iteration", "warmup_iteration",
                                                                        "begin_iteration"))))
        print("yaml", yname, "iterations", tr["max_iteration"])
    save_npz(os.path.join(HERE, "reference_sgd.npz"), out)
    print("wrote reference_sgd.npz with", len(out), "arrays")


if __name__ == "__main__":
    main()
