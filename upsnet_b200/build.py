"""Builds libupsnet_b200.so (hand-written sm_90a CUDA for H100 behind the C ABI of include/upsnet_b200.h)
in-tree with plain nvcc: no torch headers, no JIT cache.  `python -m upsnet_b200.build`."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libupsnet_b200.so")
SOURCES = ["roi_align.cu", "nms.cu", "panoptic.cu", "igemm_simt.cu", "igemm_tc.cu", "igemm_tma.cu", "dcn_win.cu", "detection.cu", "pool.cu", "post.cu", "impost.cu", "pq.cu", "sseg.cu", "cocoeval.cu", "gt_rle.cu", "combined.cu", "rpn_target.cu", "proposal_target.cu", "panoptic_loss.cu", "train_loss.cu", "labels.cu", "backward.cu", "conv_backward.cu", "sgd.cu", "group_norm.cu", "capi.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def nvcc():
    """$CUDA_HOME/bin/nvcc, else nvcc on PATH, else the default toolkit location."""
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH")):
        if home and os.path.exists(os.path.join(home, "bin", "nvcc")):
            return os.path.join(home, "bin", "nvcc")
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "include", "upsnet_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
              ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0 or verbose:
            sys.stderr.write("== %s ==\n%s\n" % (src, out))
        failed |= pr.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([nvcc()] + NVCC_FLAGS[:2] + ["-shared", "-o", LIB] + objs + ["-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
