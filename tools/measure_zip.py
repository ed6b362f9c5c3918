"""Measure the GPU zip writer (zipfile_gpu.zip_tree) against shutil.make_archive on three trees, in one process on one
GPU.

Trees, copied to a temporary directory first (so both writers read the same files from the same page cache):
numpy + numpy.libs + scipy + scipy.libs (a realistic Lambda-sized bundle), the numpy + scipy + sklearn + PIL stand-in
of BASELINE config 2, and a seeded synthetic tree of many small files (Python-like text, 200 B - 8 KB).  Per tree:

* kernels: deflate (+ compaction) and CRC-32 kernel time from CUDA events, summed over the pieces of one zip_tree
  call, and the kernel rate in GB/s of file bytes;
* end to end: wall time of zip_tree against shutil.make_archive (zlib level 6) on the same tree, both writing to the
  temporary directory.  The GPU side runs on a context created (and warmed up) before the clock starts: CUDA
  context creation is not in it, the writer's own pinned buffers and device slots are; best of --reps runs each;
* sizes: the GPU zip against make_archive's and a zlib level-1 zip of the same entries;
* files, 64 KB chunks, and chunks written stored / with the fixed code;
* the card's name and power limit, read in the same run.

    python tools/measure_zip.py [--out results/h100_zip.jsonl] [--trees numpy_scipy,config2,small_files] [--reps 3]

One JSON line per tree is printed and appended to --out.
"""
import argparse
import json
import os
import random
import shutil
import sys
import tempfile
import time
import zipfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import zipfile_gpu  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402

SITE = os.path.dirname(os.path.dirname(np.__file__))
TREES = {
    "numpy_scipy": ["numpy", "numpy.libs", "scipy", "scipy.libs"],
    "config2": ["numpy", "scipy", "sklearn", "PIL", "numpy.libs", "scipy.libs", "pillow.libs", "scikit_learn.libs"],
}


def make_tree(name, tmp):
    root = os.path.join(tmp, name)
    os.makedirs(root)
    if name in TREES:
        for d in TREES[name]:
            if os.path.exists(os.path.join(SITE, d)):
                shutil.copytree(os.path.join(SITE, d), os.path.join(root, d), symlinks=True)
        return root
    if name == "small_files":  # 30 000 files in 300 directories
        rng = random.Random(0x5EED)
        words = [bytes(rng.choices(b"abcdefghijklmnopqrstuvwxyz_", k=rng.randint(2, 10))) for _ in range(2000)]
        for d in range(300):
            dd = os.path.join(root, "pkg%03d" % d)
            os.makedirs(dd)
            for i in range(100):
                n = rng.randint(200, 8192)
                out = bytearray()
                while len(out) < n:
                    out += b"def " + rng.choice(words) + b"(" + rng.choice(words) + b"):\n    return " + rng.choice(words) + b"\n"
                with open(os.path.join(dd, "m%03d.py" % i), "wb") as f:
                    f.write(out[:n])
        return root
    raise ValueError(name)


def best(fn, reps):
    t, r = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        dt = time.perf_counter() - t0
        t = dt if t is None else min(t, dt)
    return t, r


def measure(ctx, name, tmp, gpu, reps):
    root = make_tree(name, tmp)
    gpu_path, ref_path, z1_path = (os.path.join(tmp, name + s) for s in (".gpu.zip", ".ref", ".z1.zip"))
    gpu_s, st = best(lambda: zipfile_gpu.zip_tree(root, gpu_path, ctx=ctx), reps)
    ref_s, _ = best(lambda: shutil.make_archive(ref_path, "zip", root), reps)
    with zipfile.ZipFile(z1_path, "w", compression=zipfile.ZIP_DEFLATED, compresslevel=1) as zf:
        for path, zi in zipfile_gpu.tree_entries(root):
            zf.write(path, zi.filename)
    with zipfile.ZipFile(gpu_path) as a, zipfile.ZipFile(ref_path + ".zip") as b:
        same = a.testzip() is None and [(i.filename, i.CRC, i.file_size) for i in a.infolist()] == \
            [(i.filename, i.CRC, i.file_size) for i in b.infolist()]
    gpu_b, ref_b, z1_b = (os.path.getsize(p) for p in (gpu_path, ref_path + ".zip", z1_path))
    shutil.rmtree(root)
    for p in (gpu_path, ref_path + ".zip", z1_path):
        os.remove(p)
    kernel_s = st["kernel_ms"] / 1e3
    return {
        "tree": name, "gpu": gpu, "files": st["files"], "entries": st["entries"], "in_bytes": st["in_bytes"],
        "n_chunks": st["n_chunks"], "n_stored_chunks": st["n_stored_chunks"], "n_fixed_chunks": st["n_fixed_chunks"],
        "deflate_kernel_ms": round(st["deflate_ms"], 3), "crc_kernel_ms": round(st["crc_ms"], 3),
        "kernel_GBps": round(st["in_bytes"] / kernel_s / 1e9, 3) if kernel_s else None,
        "us_per_chunk": round(st["deflate_ms"] * 1e3 / max(st["n_chunks"], 1), 2),
        "h2d_ms": round(st["h2d_ms"], 3), "d2h_ms": round(st["d2h_ms"], 3),
        "e2e_zip_tree_s": round(gpu_s, 3), "e2e_make_archive_s": round(ref_s, 3), "e2e_speedup": round(ref_s / gpu_s, 2),
        "zip_bytes_gpu": gpu_b, "zip_bytes_make_archive": ref_b, "zip_bytes_zlib1": z1_b,
        "ratio_vs_zlib6": round(gpu_b / ref_b, 4), "ratio_vs_zlib1": round(gpu_b / z1_b, 4), "entries_equal": same,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_zip.jsonl"))
    ap.add_argument("--trees", default="numpy_scipy,config2,small_files")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:
        tmp = tempfile.mkdtemp(prefix="lb2_zip_")
        try:
            warm = os.path.join(tmp, "warm")
            os.makedirs(warm)
            with open(os.path.join(warm, "w.bin"), "wb") as f:
                f.write(os.urandom(1 << 20) + bytes(1 << 20))
            zipfile_gpu.zip_tree(warm, os.path.join(tmp, "warm.zip"), ctx=ctx)   # module load, first allocations
            for name in args.trees.split(","):
                line = json.dumps(measure(ctx, name, tmp, gpu, args.reps))
                print(line, flush=True)
                os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                with open(args.out, "a") as f:
                    f.write(line + "\n")
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
