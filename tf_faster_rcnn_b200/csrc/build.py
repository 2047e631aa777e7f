"""In-tree build of libfrcnn_b200.so for sm_90a (nvcc cross-compiles without a GPU).

    python -m tf_faster_rcnn_b200.csrc.build [--force]

One object per .cu (compiled in parallel), linked with the static CUDA runtime so the library
loads on a CPU-only box for the symbol-export test."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
SOURCES = ["api.cu", "conv_gemm.cu", "simt_ops.cu", "nms.cu", "sort.cu", "attributes.cu"]
HEADERS = ["common.cuh", os.path.join("..", "..", "include", "frcnn_b200.h")]
LIB = os.path.join(PKG, "libfrcnn_b200.so")
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]


def _stale(dst, srcs):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(s) > t for s in srcs)


def build(force=False, verbose=False, watchdog=False):
    """watchdog=True builds libfrcnn_b200_wd.so (-DFRCNN_WATCHDOG: barrier waits that time out instead of hanging)."""
    obj_dir = os.path.join(HERE, "_obj_wd" if watchdog else "_obj")
    lib = LIB.replace(".so", "_wd.so") if watchdog else LIB
    flags = NVCC_FLAGS + (["-DFRCNN_WATCHDOG"] if watchdog else [])
    os.makedirs(obj_dir, exist_ok=True)
    hdrs = [os.path.join(HERE, h) for h in HEADERS]
    jobs = []
    for s in SOURCES:
        src = os.path.join(HERE, s)
        obj = os.path.join(obj_dir, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs):
            jobs.append((src, obj))

    def cc(job):
        src, obj = job
        r = subprocess.run(["nvcc"] + flags + ["-c", src, "-o", obj], capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".log", "w") as f:
            f.write(log)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, log))
        return log

    with ThreadPoolExecutor(max_workers=5) as ex:
        logs = list(ex.map(cc, jobs))
    if verbose:
        for l in logs:
            print(l)
    objs = [os.path.join(obj_dir, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(lib, objs):
        subprocess.check_call(["nvcc", "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
                               "-o", lib] + objs)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, watchdog="--watchdog" in sys.argv))
