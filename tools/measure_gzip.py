"""Measure the GPU gzip writer against zlib on three trees, in one process on one GPU.

Trees: site-packages numpy + numpy.libs + scipy + scipy.libs, torch/lib, and a seeded synthetic corpus
(lambdipy_b200.corpus: ELF files with random payload, so most chunks take the stored path).  Per tree:

* kernels: deflate (+ compaction) and CRC-32 kernel time from CUDA events, over the tar stream held in
  memory and fed in 64 MB pieces, and kernel GB/s of input;
* end to end: wall time of tarball.gzip_tarball (the mirror's body) against stdlib
  `tarfile.open(path, "w:gz")` with the same add loop, both writing to a temporary directory.  The GPU side
  runs on a context created (and warmed up) before the clock starts: CUDA context creation is not in it, the
  writer's own pinned buffers and device slots are;
* ratios: compressed / tar bytes for the GPU, zlib level 1 and zlib level 9 (the stdlib tarball's size);
* the card's name and power limit, read in the same run.

    python tools/measure_gzip.py [--out results/h100_gzip.jsonl] [--trees numpy_scipy,torch_lib,synthetic]

One JSON line per tree is printed and appended to --out.
"""
import argparse
import io
import json
import os
import shutil
import subprocess
import sys
import tarfile
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import tarball  # noqa: E402

SITE = os.path.dirname(os.path.dirname(np.__file__))


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
    except OSError:
        return "unknown"
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def tree_sources(name, tmp):
    if name == "numpy_scipy":
        return [os.path.join(SITE, d) for d in ("numpy", "numpy.libs", "scipy", "scipy.libs") if os.path.exists(os.path.join(SITE, d))]
    if name == "torch_lib":
        import torch
        return [os.path.join(os.path.dirname(torch.__file__), "lib")]
    if name == "synthetic":
        from lambdipy_b200.corpus import Corpus
        corpus = Corpus(64, seed=0x6219, max_size=64 << 20)   # 285 MB
        d = os.path.join(tmp, "synthetic")
        os.makedirs(d)
        for i in range(len(corpus)):
            with open(os.path.join(d, "lib%03d.so" % i), "wb") as f:
                f.write(corpus.materialize(i))
        return [d]
    raise ValueError(name)


def tar_stream(srcs):
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        for p in srcs:
            tar.add(p, arcname=os.path.basename(p))
    return buf.getvalue()


def gpu_deflate(ctx, data, piece=64 << 20):
    """the tar stream through lb2_gzip_* with two pieces in flight; returns (DEFLATE bytes, stats, wall s)"""
    import ctypes as C
    lib = ctx.lib
    g = C.c_void_p()
    ctx.check(lib.lb2_gzip_create(ctx.h, 0, C.byref(g)))
    bufs = [ctx.pinned_alloc(piece) for _ in range(2)]
    cap = N.gzip_bound(piece)
    out = ctx.pinned_alloc(cap)
    n = C.c_uint64()
    total, in_flight = 0, 0
    try:
        t0 = time.perf_counter()
        for k, off in enumerate(range(0, len(data), piece)):
            if in_flight == 2:
                ctx.check(lib.lb2_gzip_collect(g, out, cap, C.byref(n)))
                total += n.value
                in_flight -= 1
            m = min(piece, len(data) - off)
            C.memmove(bufs[k & 1], data[off:off + m], m)
            ctx.check(lib.lb2_gzip_submit(g, bufs[k & 1], m))
            in_flight += 1
        while in_flight:
            ctx.check(lib.lb2_gzip_collect(g, out, cap, C.byref(n)))
            total += n.value
            in_flight -= 1
        crc, isize, st = C.c_uint32(), C.c_uint64(), N.GzipStats()
        ctx.check(lib.lb2_gzip_finish(g, out, cap, C.byref(n), C.byref(crc), C.byref(isize), C.byref(st)))
        wall = time.perf_counter() - t0
        total += n.value
    finally:
        lib.lb2_gzip_destroy(g)
        for b in bufs:
            ctx.pinned_free(b)
        ctx.pinned_free(out)
    assert crc.value == zlib.crc32(data) and isize.value == len(data)
    return total, st.as_dict(), wall


def measure(ctx, name, tmp, gpu):
    srcs = tree_sources(name, tmp)
    data = tar_stream(srcs)
    body, st, wall = gpu_deflate(ctx, data)
    kernel_s = (st["deflate_ms"] + st["crc_ms"]) / 1e3
    t0 = time.perf_counter()
    lvl1 = len(zlib.compress(data, 1))
    z1_s = time.perf_counter() - t0

    gpu_path, ref_path = os.path.join(tmp, name + ".gpu.tar.gz"), os.path.join(tmp, name + ".ref.tar.gz")
    t0 = time.perf_counter()
    tarball.gzip_tarball(srcs, gpu_path, ctx=ctx)
    gpu_e2e = time.perf_counter() - t0
    t0 = time.perf_counter()
    with tarfile.open(ref_path, "w:gz") as tar:
        for p in srcs:
            tar.add(p, arcname=os.path.basename(p))
    ref_e2e = time.perf_counter() - t0
    import gzip
    with gzip.open(gpu_path, "rb") as a, gzip.open(ref_path, "rb") as b:
        same = a.read() == b.read()
    gpu_file, ref_file = os.path.getsize(gpu_path), os.path.getsize(ref_path)
    os.remove(gpu_path)
    os.remove(ref_path)
    return {
        "tree": name, "sources": [os.path.relpath(p, SITE) if p.startswith(SITE) else os.path.basename(p) for p in srcs],
        "tar_bytes": len(data), "gpu": gpu,
        "deflate_kernel_ms": round(st["deflate_ms"], 3), "crc_kernel_ms": round(st["crc_ms"], 3),
        "kernel_GBps": round(len(data) / kernel_s / 1e9, 3),
        "h2d_ms": round(st["h2d_ms"], 3), "d2h_ms": round(st["d2h_ms"], 3),
        "gpu_stream_wall_s": round(wall, 3),
        "n_chunks": st["n_chunks"], "n_stored_chunks": st["n_stored_chunks"], "n_fixed_chunks": st["n_fixed_chunks"],
        "ratio_gpu": round(body / len(data), 4), "ratio_zlib1": round(lvl1 / len(data), 4),
        "ratio_zlib9": round(ref_file / len(data), 4), "zlib1_s": round(z1_s, 3),
        "e2e_gpu_mirror_s": round(gpu_e2e, 3), "e2e_tarfile_w_gz_s": round(ref_e2e, 3),
        "e2e_speedup": round(ref_e2e / gpu_e2e, 2), "gpu_file_bytes": gpu_file, "ref_file_bytes": ref_file,
        "tar_streams_equal": same,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_gzip.jsonl"))
    ap.add_argument("--trees", default="numpy_scipy,torch_lib,synthetic")
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:
        gpu_deflate(ctx, os.urandom(1 << 20) + bytes(1 << 20))   # module load, first allocations
        tmp = tempfile.mkdtemp(prefix="lb2_gzip_")
        try:
            for name in args.trees.split(","):
                rec = measure(ctx, name, tmp, gpu)
                line = json.dumps(rec)
                print(line, flush=True)
                os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                with open(args.out, "a") as f:
                    f.write(line + "\n")
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
