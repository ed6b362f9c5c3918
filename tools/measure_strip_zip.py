"""strip_zip (inflate, strip and deflate chained on the GPU) against the three passes it replaces.

For each tree -- numpy + numpy.libs + scipy + scipy.libs (a realistic Lambda bundle) and torch/lib (few, very large
members) -- the tree is zipped by shutil.make_archive, and that zip is then stripped twice, end to end:
  - by zipfile_gpu.strip_zip, on a context created before the clock starts;
  - by ZipFile.extractall, the reference's `find -name "*.so" | xargs strip` and shutil.make_archive, on the same
    disk.
The two results are compared member by member (the same names, and every member's decompressed bytes).  The kernel
times of the three engines (CUDA events), the bytes that crossed the bus, the card name and its power limit are read
in the same process.  One JSON line per tree is printed and appended to --out.

    python tools/measure_strip_zip.py [--out results/h100_strip_zip.jsonl] [--trees numpy_scipy,torch_lib] [--reps 1]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import zipfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import zipfile_gpu  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402
from measure_unzip import tree_root  # noqa: E402
from measure_zip import best  # noqa: E402


def three_passes(src, tmp):
    """extractall + the reference's strip line + make_archive; returns (the zip, seconds of each pass)"""
    d = os.path.join(tmp, "passes")
    shutil.rmtree(d, ignore_errors=True)
    t0 = time.perf_counter()
    with zipfile.ZipFile(src) as zf:
        zf.extractall(d)
    t1 = time.perf_counter()
    rc = subprocess.run('find %s/ -name "*.so" | xargs strip' % d, shell=True).returncode
    t2 = time.perf_counter()
    out = shutil.make_archive(os.path.join(tmp, "passes_out"), "zip", d)
    t3 = time.perf_counter()
    shutil.rmtree(d)
    if rc:
        raise RuntimeError("the reference's strip line exited %d" % rc)
    return out, (t1 - t0, t2 - t1, t3 - t2)


def same_members(a_path, b_path):
    """the same names (make_archive orders them by its own walk) and, name by name, the same bytes"""
    with zipfile.ZipFile(a_path) as a, zipfile.ZipFile(b_path) as b:
        if sorted(a.namelist()) != sorted(b.namelist()) or len(set(a.namelist())) != len(a.namelist()):
            return False
        return all(a.getinfo(n).is_dir() or (a.getinfo(n).CRC == b.getinfo(n).CRC and a.read(n) == b.read(n))
                   for n in b.namelist())


def measure(ctx, name, src, tmp, gpu, reps):
    dst = os.path.join(tmp, name + "_stripped.zip")
    gpu_s, st = best(lambda: zipfile_gpu.strip_zip(src, dst, ctx=ctx), reps)
    ref_s, (ref_zip, passes) = best(lambda: three_passes(src, tmp), reps)
    t0 = time.perf_counter()
    identical = same_members(ref_zip, dst)
    cmp_s = time.perf_counter() - t0
    ref_bytes = os.path.getsize(ref_zip)
    os.remove(ref_zip)
    os.remove(dst)
    uz, sp, df = st["unzip"], st["strip"], st["deflate"]
    return {
        "tree": name, "gpu": gpu, "members": st["members"], "selected": st["selected"], "gpu_members": st["gpu"],
        "fallback": st["fallback"], "skipped": st["skipped"], "so_bytes_in": st["in_bytes"], "so_bytes_out": st["out_bytes"],
        "src_zip_bytes": st["src_zip_bytes"], "zip_bytes": st["zip_bytes"], "three_pass_zip_bytes": ref_bytes,
        "uploaded_bytes": st["uploaded_bytes"], "downloaded_bytes": st["downloaded_bytes"],
        "unzip_kernel_ms": round(uz["kernel_ms"], 3), "plan_ms": round(sp["plan_ms"], 3), "compact_ms": round(sp["compact_ms"], 3),
        "gather_ms": round(df["h2d_ms"], 3), "deflate_ms": round(df["deflate_ms"], 3), "deflate_crc_ms": round(df["crc_ms"], 3),
        "kernel_ms": round(st["kernel_ms"], 3), "e2e_strip_zip_s": round(gpu_s, 3), "e2e_three_passes_s": round(ref_s, 3),
        "extractall_s": round(passes[0], 3), "find_xargs_strip_s": round(passes[1], 3), "make_archive_s": round(passes[2], 3),
        "speedup": round(ref_s / gpu_s, 2), "members_identical": identical, "compare_s": round(cmp_s, 2), "reps": reps,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_strip_zip.jsonl"))
    ap.add_argument("--trees", default="numpy_scipy,torch_lib")
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:   # no device: this raises, nothing is timed
        tmp = tempfile.mkdtemp(prefix="lb2_strip_zip_")
        try:
            warm = os.path.join(tmp, "warm.zip")   # module load and first allocations of the three engines
            with zipfile.ZipFile(warm, "w", zipfile.ZIP_DEFLATED) as zf:
                zf.write(os.path.join(ROOT, "tests", "golden", "cxx_g.in.bin"), "warm/cxx_g.so")
            zipfile_gpu.strip_zip(warm, os.path.join(tmp, "warm_out.zip"), ctx=ctx)
            for name in args.trees.split(","):
                root = tree_root(name, tmp)
                src = shutil.make_archive(os.path.join(tmp, name + "_src"), "zip", root)
                shutil.rmtree(root)
                line = json.dumps(measure(ctx, name, src, tmp, gpu, args.reps))
                print(line, flush=True)
                os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                with open(args.out, "a") as f:
                    f.write(line + "\n")
                os.remove(src)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
