"""Measure the seek table: the gzip writer and reader with and without it, on the trees of tools/measure_gzip.py.

Per tree (site-packages numpy + numpy.libs + scipy + scipy.libs, torch/lib), the tarball is written by
tarball.gzip_tarball with and without seek_table, the two runs alternating, --reps times each, on a context created
(and warmed up) before any clock starts.  Recorded per variant, as the median over the repetitions:

* writer: kernel time (deflate + CRC-32, CUDA events), wall time and file size;
* reader: the kernels (find / count / decode / resolve / CRC-32, CUDA events), spans, count rounds, and whether the
  table was used, from one read of the file through tarball.inflate_members;
* end to end: tarball.extract_tarball and tarball.strip_tarball of the file (host clock);
* the zip side, on the tree's first directory (numpy, torch/lib): zipfile_gpu.zip_tree with and without seek_table,
  then extract_zip, testzip and strip_zip of each zip, with the zip reader's kernel times and table counts;
* the card's name, power limit and maximum SM clock, read in the same run.

    python tools/measure_seek_table.py [--out results/h100_seek_table.jsonl] [--trees numpy_scipy,torch_lib] [--reps 3]

One JSON line per tree is printed and appended to --out.
"""
import argparse
import ctypes as C
import json
import os
import shutil
import statistics
import sys
import tarfile
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lambdipy_b200 import seek_table as ST  # noqa: E402
from lambdipy_b200 import tarball, zipfile_gpu  # noqa: E402
from lambdipy_b200.seek_table import seek_kw  # noqa: E402
from measure_gzip import gpu_info, tree_sources  # noqa: E402

KERNELS = ("find_ms", "count_ms", "decode_ms", "resolve_ms", "crc_ms")


def read_stats(ctx, path):
    d = C.c_void_p()
    ctx.check(ctx.lib.lb2_inflate_create(ctx.h, 0, C.byref(d)))
    stats, counts = {}, {}
    try:
        def on_member(isize, last, st):
            for k, v in st.as_dict().items():
                stats[k] = stats.get(k, 0) + v
        t0 = time.perf_counter()
        tarball.inflate_members(ctx, d, path, on_member, counts)
        wall = time.perf_counter() - t0
    finally:
        ctx.lib.lb2_inflate_destroy(d)
    out = {k: round(stats.get(k, 0.0), 2) for k in KERNELS}
    out.update(kernel_ms=round(sum(stats.get(k, 0.0) for k in KERNELS), 2), n_spans=stats.get("n_spans", 0),
               n_rounds=stats.get("n_rounds", 0), seek_table=counts.get("seek_table", 0),
               seek_table_refused=counts.get("seek_table_refused", 0), wall_s=round(wall, 3))
    return out


def one(ctx, srcs, tmp, seek):
    path = os.path.join(tmp, "seek" if seek else "plain", "pkg.tar.gz")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    t0 = time.perf_counter()
    with tarball.GpuGzipFile(path, ctx=ctx, seek_table=seek) as gz:
        with tarfile.open(name=path, mode="w", fileobj=gz) as tar:
            for p in srcs:
                tar.add(p, arcname=os.path.basename(p))
    write_s = time.perf_counter() - t0
    st = gz.stats
    rec = {"write_s": write_s, "write_kernel_ms": st["deflate_ms"] + st["crc_ms"], "bytes": os.path.getsize(path)}
    rec["read"] = read_stats(ctx, path)
    out = os.path.join(tmp, "x")
    t0 = time.perf_counter()
    tarball.extract_tarball(path, out, ctx=ctx)
    rec["extract_s"] = time.perf_counter() - t0
    shutil.rmtree(out)
    dst = os.path.join(tmp, "stripped.tar.gz")
    t0 = time.perf_counter()
    s = tarball.strip_tarball(path, dst, ctx=ctx, seek_table=seek)
    rec["strip_s"] = time.perf_counter() - t0
    rec["strip_inflate_kernel_ms"] = s["inflate"]["kernel_ms"]
    rec["strip_kernel_ms"] = s["kernel_ms"]
    os.unlink(dst)
    zpath = os.path.join(tmp, "seek" if seek else "plain", "t.zip")
    zipfile_gpu.zip_tree(srcs[0], zpath, ctx=ctx, **seek_kw(seek))
    rec["zip_bytes"] = os.path.getsize(zpath)
    for what, fn in (("extract_zip", lambda: zipfile_gpu.extract_zip(zpath, out, ctx=ctx)),
                     ("testzip", lambda: {"bad": zipfile_gpu.testzip(zpath, ctx=ctx)}),
                     ("strip_zip", lambda: zipfile_gpu.strip_zip(zpath, dst + ".zip", ctx=ctx, **seek_kw(seek)))):
        t0 = time.perf_counter()
        r = fn()
        rec[what + "_s"] = time.perf_counter() - t0
        if what == "extract_zip":
            rec["unzip_kernel_ms"] = r["kernel_ms"]
            rec["unzip_read"] = {k: round(r.get(k, 0), 2) for k in KERNELS + ("small_ms", "copy_ms", "n_spans",
                                                                                 "n_small", "n_large", "seek_table",
                                                                                 "seek_table_refused")}
            shutil.rmtree(out, ignore_errors=True)
    os.unlink(dst + ".zip")
    if seek:
        with open(path, "rb") as f:
            raw = f.read()
        off, entries = ST.gzip_tail(raw)
        rec["entries"], rec["table_bytes"] = len(entries), len(raw) - off
    return rec


def median(recs, key):
    return round(statistics.median(r[key] for r in recs), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_seek_table.jsonl"))
    ap.add_argument("--trees", default="numpy_scipy,torch_lib")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from lambdipy_b200 import _native as N
    ctx = N.Context(0)
    warm = tempfile.mkdtemp()
    try:   # module loads and first launches of every kernel, before any clock
        with open(os.path.join(warm, "w.bin"), "wb") as f:
            f.write(os.urandom(1 << 20) * 3)
        one(ctx, [os.path.join(warm, "w.bin")], warm, True)
    finally:
        shutil.rmtree(warm)
    card = gpu_info()
    for name in args.trees.split(","):
        tmp = tempfile.mkdtemp(prefix="seek_")
        try:
            srcs = tree_sources(name, tmp)
            runs = {False: [], True: []}
            for _ in range(args.reps):
                for seek in (False, True):
                    runs[seek].append(one(ctx, srcs, tmp, seek))
            rec = {"tree": name, "gpu": card, "reps": args.reps}
            for seek, key in ((False, "no_table"), (True, "table")):
                r = runs[seek]
                rec[key] = {k: median(r, k) for k in ("write_s", "write_kernel_ms", "bytes", "extract_s", "strip_s",
                                                     "strip_inflate_kernel_ms", "strip_kernel_ms", "zip_bytes",
                                                     "extract_zip_s", "testzip_s", "strip_zip_s", "unzip_kernel_ms")}
                rec[key]["read"] = {k: round(statistics.median(x["read"][k] for x in r), 3) for k in r[0]["read"]}
                rec[key]["unzip_read"] = {k: round(statistics.median(x["unzip_read"][k] for x in r), 3)
                                          for k in r[0]["unzip_read"]}
                rec[key]["read_kernel_ms_all"] = [x["read"]["kernel_ms"] for x in r]
                rec[key]["extract_s_all"] = [round(x["extract_s"], 3) for x in r]
                if seek:
                    rec[key]["entries"], rec[key]["table_bytes"] = r[-1]["entries"], r[-1]["table_bytes"]
            line = json.dumps(rec)
            print(line, flush=True)
            os.makedirs(os.path.dirname(args.out), exist_ok=True)
            with open(args.out, "a") as f:
                f.write(line + "\n")
        finally:
            shutil.rmtree(tmp)
    ctx.close()


if __name__ == "__main__":
    main()
