"""In-tree build of the sm_90a shared library (no JIT cache: the .so must travel with the repo snapshot)."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libmeshdiff_b200.so")
SOURCES = ["gemm_host.cu", "wgrad_host.cu", "elementwise.cu", "backward.cu", "unet.cu", "unet_train.cu", "marching_tets.cu", "mesh_ops.cu", "train_ops.cu", "pc_metrics.cu", "emd.cu", "likelihood.cu", "raster.cu", "fit.cu", "depth_partial.cu", "interp.cu", "lfd.cu", "repaint.cu", "distill.cu", "api.cu"]
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH_FLAGS + [
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
    "-Xptxas", "-v",  # the per-kernel report is where ptxas says it had to serialise wgmma (checked below)
]
# ptxas reports that make a wgmma kernel issue one MMA at a time (it waits for each to finish before the next): a build that
# would silently lose the MMA pipelining fails instead
SERIALISED_WGMMA = ("C7510", "C7520")
# Kernels that must keep every value in registers. Their shared-memory rings leave L1 about 28 KB, so a stack frame (an
# array indexed by a lane-dependent value, which ptxas does not count as a spill) or a spill goes to L2, on the
# critical path of the epilogue or the MMA loop. No kernel here needs a stack.
NO_STACK_KERNELS = ("gemm_tc_kernel", "wgrad_tc_kernel")
_PROPS = re.compile(r"Function properties for (\S+)")
_FRAME = re.compile(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")


def local_memory_violations(ptxas_report):
    """Lines of a `-Xptxas -v` report where a NO_STACK_KERNELS function has a stack frame or spills."""
    bad, fn = [], None
    for line in ptxas_report.splitlines():
        m = _PROPS.search(line)
        if m:
            fn = m.group(1)
            continue
        m = _FRAME.search(line)
        if m and fn and any(k in fn for k in NO_STACK_KERNELS) and any(int(g) for g in m.groups()):
            bad.append(f"{fn}: {line.strip()}")
        fn = None
    return bad


def _newest_mtime(paths):
    return max(os.path.getmtime(p) for p in paths)


def build(force=False, verbose=False):
    """Compiles the library unless it is newer than every source. Serialised by a file lock: under torchrun every rank may
    find the library missing at the same moment; one compiles, the others wait and then see an up-to-date file."""
    import fcntl
    os.makedirs(LIBDIR, exist_ok=True)
    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose):
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "meshdiff_b200.h")]
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_mtime(deps):
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    for s in srcs:
        o = os.path.join(LIBDIR, os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        out = out.decode()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
        serialised = [line for line in out.splitlines() if any(code in line for code in SERIALISED_WGMMA)]
        if serialised:
            raise RuntimeError("ptxas serialised wgmma in " + cmd[-3] + ":\n" + "\n".join(serialised))
        local = local_memory_violations(out)
        if local:
            raise RuntimeError("local memory in a register-only kernel of " + cmd[-3] + ":\n" + "\n".join(local))
    cmd = [nvcc] + ARCH_FLAGS + ["-shared", "-o", LIB] + objs + ["-lcudart", "-ldl"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
