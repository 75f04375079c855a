"""In-tree build of the CUDA C-ABI library (sm_90a only, no JIT cache)."""
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB = os.path.join(CSRC, "libb200ps.so")
SOURCES = ["b200ps.cu", "deepfm_tower.cu", "deepfm_tower_mma.cu", "deepfm_tower2.cu", "dcn_tower.cu", "xdeepfm_cin.cu",
           "feature_ids.cu", "census_tower.cu", "frappe_tower.cu", "eval_metrics.cu", "fc_dnn_tower.cu",
           "census_sqlflow_tower.cu", "deepctr_wdl_tower.cu", "deepctr_deepfm_tower.cu"]
HEADERS = ["ps_kernels.cuh", "ps_types.cuh", "ps_exchange.cuh", "ps_flat.cuh", "ps_unique.cuh", "deepfm_common.cuh",
           "tile_tower.cuh", "mma_tf32.cuh", "xdeepfm.cuh", "launch.cuh", "census_tower.cuh", "deepctr_dnn.cuh",
           os.path.join("..", "..", "include", "b200ps.h"),
           os.path.join("..", "..", "include", "b200_deepfm.h"),
           os.path.join("..", "..", "include", "b200_features.h"),
           os.path.join("..", "..", "include", "b200_census.h"),
           os.path.join("..", "..", "include", "b200_frappe.h"),
           os.path.join("..", "..", "include", "b200_metrics.h"),
           os.path.join("..", "..", "include", "b200_fc_dnn.h"),
           os.path.join("..", "..", "include", "b200_census_sqlflow.h"),
           os.path.join("..", "..", "include", "b200_deepctr_wdl.h"),
           os.path.join("..", "..", "include", "b200_deepctr_deepfm.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


STAMP = LIB + ".sources.sha256"


def _sources_digest():
    import hashlib

    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode() + b"\0" + fh.read() + b"\0")
    return h.hexdigest()


def _stale():
    """The library is current iff the digest of the sources it was built from (a sidecar file that travels
    with it) equals the digest of the sources in the tree -- file times do not survive a snapshot / checkout."""
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as fh:
        return fh.read().strip() != _sources_digest()


def build(force=False, verbose=False):
    """Compile elasticdl_b200/csrc/*.cu -> libb200ps.so with nvcc (cross-compiles without a GPU)."""
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    # rank-per-GPU runs import this module in every rank at once: one builder at a time (file lock),
    # and the library appears atomically (compile to a temporary name, then rename) so that no
    # process can dlopen a half-written file
    import fcntl

    with open(os.path.join(CSRC, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not _stale():  # another rank built it while we waited
                return LIB
            tmp = LIB + ".tmp.%d" % os.getpid()
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + SOURCES
            digest = _sources_digest()
            subprocess.check_call(cmd, cwd=CSRC)
            os.replace(tmp, LIB)
            with open(STAMP + ".tmp", "w") as fh:
                fh.write(digest + "\n")
            os.replace(STAMP + ".tmp", STAMP)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
