"""Where the implicit-GEMM epilogue's time goes: globaltimer stamps from an instrumented build of the library.

Compiles the library with -DMDB_EPI_TRACE into --lib-dir (once; the default build has no trace code), runs res64 forwards
at batch 32 with synthetic weights in each requested operand mode, and reads the stamps the first 64 tiles of the first
16 CTAs of every launch wrote (see gemm_tc.cuh, MDB_STAMP). For the 64^3 halo convolutions (65 536 work items of 128
columns, three k-steps per entry) it prints the mean time per tile from the last wgmma_wait<0> to:

  staged   round 0's accumulators staged (named barrier passed)
  round0   round 0's chunks done (TMA epilogue: its output store issued)
  round1   round 1 staged and its chunks done
  stats    the GroupNorm statistics atomics done
  next     the next tile's first k-step has its operands (the end of the tile's fixed cost)

--per-thread also times the per-thread stores and loads on the same launches (MDB_EPI_TRACE_PER_THREAD, read by the
instrumented build only), in the same process. The globaltimer ticks in steps of about a microsecond on some parts;
the means are over thousands of tiles. The card's name, power limit and SM clock are read in the same process.

    python tools/epi_trace.py --precision bf16x3 bf16 --per-thread [--json out.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

PHASES = ("staged", "round0", "round1", "stats", "next")


def build_traced(lib_dir):
    """The instrumented library in lib_dir (compiled unless it is newer than every source)."""
    from meshdiffusion_b200 import build as B
    lib = os.path.join(lib_dir, "libmeshdiff_b200.so")
    deps = [os.path.join(B.CSRC, f) for f in os.listdir(B.CSRC)] + [os.path.join(ROOT, "include", "meshdiff_b200.h")]
    if os.path.exists(lib) and os.path.getmtime(lib) >= max(os.path.getmtime(d) for d in deps):
        return lib
    os.makedirs(lib_dir, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs, procs = [], []
    for s in B.SOURCES:
        o = os.path.join(lib_dir, s[:-3] + ".o")
        objs.append(o)
        cmd = [nvcc] + B.NVCC_FLAGS + ["-DMDB_EPI_TRACE", "-c", os.path.join(B.CSRC, s), "-o", o]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
    for p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise SystemExit("nvcc failed")
    subprocess.check_call([nvcc] + B.ARCH_FLAGS + ["-shared", "-o", lib] + objs + ["-lcudart", "-ldl"])
    return lib


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def read_traces(L):
    ctas, tiles, stamps = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    L.mdb_epi_trace_dims(ctypes.byref(ctas), ctypes.byref(tiles), ctypes.byref(stamps))
    shape = (ctas.value, tiles.value, stamps.value)
    buf = (ctypes.c_ulonglong * int(np.prod(shape)))()
    name = ctypes.create_string_buffer(256)
    out, i = {}, 0
    while True:
        n = L.mdb_epi_trace_read(i, name, 256, buf)
        if n == -1:
            return out
        if n < 0:
            raise RuntimeError("mdb_epi_trace_read failed")
        out[name.value.decode()] = np.ctypeslib.as_array(buf).reshape(shape).astype(np.int64).copy()
        i += 1


def phases(tr):
    """[tiles, 5] nanoseconds per phase of every traced tile whose stamps and next tile's stamp 5 are all present."""
    s = tr[:, :-1, :]
    nxt = tr[:, 1:, 5]
    ok = (s[..., :5] > 0).all(-1) & (nxt > 0)
    t = np.stack([s[..., 1] - s[..., 0], s[..., 2] - s[..., 1], s[..., 3] - s[..., 2], s[..., 4] - s[..., 3],
                  nxt - s[..., 4]], -1)
    return t[ok]


def run(precision, batch=32):
    import torch
    import bench
    dev = torch.device("cuda:0")
    _, model = bench.build_model(precision, batch, dev, 64)
    net = model.module
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(batch, 4, 64, 64, 64, device=dev, generator=g)
    labels = torch.full((batch,), 500.0, device=dev)
    with torch.no_grad():
        for _ in range(2):
            model(x, labels)
    torch.cuda.synchronize()
    from meshdiffusion_b200 import _native
    traces = read_traces(_native.lib())
    names = [n for n, _, _ in net.gemm_ops()]
    group = [n for n, (work, splits, _, entry_k, block_n) in zip(names, net.gemm_tiles())
             if work == 65536 and splits == 1 and entry_k == 3 and block_n == 128]
    t = np.concatenate([phases(traces[n]) for n in group if n in traces]) / 1e3
    net.release_engine()
    del model
    torch.cuda.empty_cache()
    return {"precision": precision, "launches": len(group), "tiles": int(t.shape[0]),
            "us": {k: float(v) for k, v in zip(PHASES, t.mean(0))}, "total_us": float(t.sum(1).mean()), "card": card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", nargs="+", default=["bf16x3", "bf16"])
    ap.add_argument("--per-thread", action="store_true", help="also trace the per-thread stores on the same launches")
    ap.add_argument("--lib-dir", default=os.path.join(ROOT, "meshdiffusion_b200", "lib", "epi_trace"))
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from meshdiffusion_b200 import _native
    _native.LIB_PATH = build_traced(a.lib_dir)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("epi_trace needs a GPU")
    rows = []
    for prec in a.precision:
        for per_thread in ([False, True] if a.per_thread else [False]):
            if per_thread:
                os.environ["MDB_EPI_TRACE_PER_THREAD"] = "1"
            else:
                os.environ.pop("MDB_EPI_TRACE_PER_THREAD", None)
            r = run(prec)
            r["epilogue"] = "per-thread" if per_thread else "default"
            rows.append(r)
            ph = "  ".join(f"{k} {r['us'][k]:.2f}" for k in PHASES)
            print(f"{prec:<7} {r['epilogue']:<11} {r['launches']} launches, {r['tiles']} tiles: {ph}  "
                  f"total {r['total_us']:.2f} us  [{r['card']}]", flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
