"""Measure the GPU gzip reader against zlib and `tarfile "r:gz"` on three trees, in one process on one GPU.

Trees as in tools/measure_gzip.py: site-packages numpy + numpy.libs + scipy + scipy.libs, torch/lib, and a seeded
synthetic corpus.  Each tree's tarball is written twice: by stdlib `tarfile "w:gz"` (zlib level 9, like the
published assets) and by tarball.gzip_tarball.  Per tarball:

* kernels: find / count / decode / resolve / CRC-32 times from CUDA events, and the kernel rate in GB/s of output;
* the chain: n_spans, n_rounds, n_rejected, n_absorbed;
* one-core zlib.decompress time of the same body;
* end to end: tarball.extract_tarball against `tarfile.open(p, "r:gz").extractall(d)` on the same host, the GPU
  side on a context created (and warmed up) before the clock starts; and whether the two trees are identical;
* the card's name, power limit and maximum SM clock, read in the same run.

    python tools/measure_gunzip.py [--out results/h100_gunzip.jsonl] [--trees numpy_scipy,torch_lib,synthetic]

One JSON line per tarball is printed and appended to --out.
"""
import argparse
import ctypes as C
import filecmp
import json
import os
import shutil
import sys
import tarfile
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import tarball  # noqa: E402
from measure_gzip import SITE, gpu_info, tree_sources  # noqa: E402


def gpu_inflate(ctx, body):
    d = C.c_void_p()
    ctx.check(ctx.lib.lb2_inflate_create(ctx.h, 0, C.byref(d)))
    h = ctx.pinned_alloc(len(body))
    try:
        C.memmove(h, body, len(body))
        n, st = C.c_uint64(), N.InflateStats()
        t0 = time.perf_counter()
        ctx.check(ctx.lib.lb2_inflate_run(d, h, len(body), C.byref(n), C.byref(st)))
        wall = time.perf_counter() - t0
        return n.value, st.as_dict(), wall
    finally:
        ctx.lib.lb2_inflate_destroy(d)
        ctx.pinned_free(h)


def same_tree(a, b):
    for dp, dns, fns in os.walk(a):
        for n in dns + fns:
            p = os.path.join(dp, n)
            q = os.path.join(b, os.path.relpath(p, a))
            if not os.path.lexists(q) or os.path.islink(p) != os.path.islink(q):
                return False
            sp, sq = os.lstat(p), os.lstat(q)
            if sp.st_mode != sq.st_mode or int(sp.st_mtime) != int(sq.st_mtime):
                return False
            if os.path.islink(p):
                if os.readlink(p) != os.readlink(q):
                    return False
            elif os.path.isfile(p) and not filecmp.cmp(p, q, shallow=False):
                return False
    return sum(len(d) + len(f) for _, d, f in os.walk(a)) == sum(len(d) + len(f) for _, d, f in os.walk(b))


def measure(ctx, name, writer, srcs, tmp, gpu):
    path = os.path.join(tmp, "%s.%s.tar.gz" % (name, writer))
    if writer == "tarfile_w_gz_9":
        with tarfile.open(path, "w:gz") as tar:
            for p in srcs:
                tar.add(p, arcname=os.path.basename(p))
    else:
        tarball.gzip_tarball(srcs, path, ctx=ctx)
    with open(path, "rb") as f:
        raw = f.read()
    flags, p = raw[3], 10
    if flags & tarball.FNAME:
        p = raw.index(b"\0", p) + 1
    body = raw[p:]
    out_n, st, wall = gpu_inflate(ctx, body)
    t0 = time.perf_counter()
    zlen = len(zlib.decompressobj(-15).decompress(body))
    z_s = time.perf_counter() - t0
    assert zlen == out_n
    kernel_ms = st["find_ms"] + st["count_ms"] + st["decode_ms"] + st["resolve_ms"] + st["crc_ms"]
    mine, ref = os.path.join(tmp, "x_mine"), os.path.join(tmp, "x_ref")
    t0 = time.perf_counter()
    tarball.extract_tarball(path, mine, ctx)
    gpu_e2e = time.perf_counter() - t0
    t0 = time.perf_counter()
    with tarfile.open(path, "r:gz") as tar:
        tar.extractall(ref)
    ref_e2e = time.perf_counter() - t0
    same = same_tree(mine, ref)
    shutil.rmtree(mine)
    shutil.rmtree(ref)
    os.remove(path)
    nominal = (len(body) + (128 << 10) - 1) // (128 << 10)
    return {
        "tree": name, "writer": writer, "gpu": gpu, "gz_bytes": len(raw), "tar_bytes": out_n,
        **{k: round(st[k], 3) for k in ("find_ms", "count_ms", "decode_ms", "resolve_ms", "crc_ms", "h2d_ms")},
        "kernel_ms": round(kernel_ms, 3), "kernel_GBps_out": round(out_n / kernel_ms / 1e6, 3),
        "run_wall_s": round(wall, 3), "nominal_spans": nominal,
        **{k: st[k] for k in ("n_spans", "n_rounds", "n_rejected", "n_absorbed")},
        "zlib_decompress_s": round(z_s, 3), "e2e_extract_tarball_s": round(gpu_e2e, 3),
        "e2e_tarfile_r_gz_s": round(ref_e2e, 3), "e2e_speedup": round(ref_e2e / gpu_e2e, 2), "trees_identical": same,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_gunzip.jsonl"))
    ap.add_argument("--trees", default="numpy_scipy,torch_lib,synthetic")
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:
        gpu_inflate(ctx, zlib.compress(os.urandom(1 << 20) + bytes(1 << 20), 9)[2:-4])   # module load, allocations
        tmp = tempfile.mkdtemp(prefix="lb2_gunzip_")
        try:
            for name in args.trees.split(","):
                srcs = tree_sources(name, tmp)
                for writer in ("tarfile_w_gz_9", "gzip_tarball"):
                    rec = measure(ctx, name, writer, srcs, tmp, gpu)
                    line = json.dumps(rec)
                    print(line, flush=True)
                    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                    with open(args.out, "a") as f:
                        f.write(line + "\n")
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
