"""Zip reader on the GPU (zipfile_gpu.extract_zip / testzip, lb2_unzip_*) against ZipFile.extractall / testzip.

Trees: numpy + numpy.libs + scipy + scipy.libs (a realistic Lambda bundle), torch/lib (few, very large members) and
30 000 small generated files.  Each tree is zipped twice, by shutil.make_archive (zlib level 6) and by zip_tree (the
GPU writer), and each zip is then
  - extracted by extract_zip and by ZipFile.extractall, end to end, into fresh directories on the same disk;
  - tested by testzip and by ZipFile.testzip, end to end;
  - its two extracted trees compared file by file;
with the kernel times of the reader (CUDA events) from the extract_zip run.  The card name and power limit are read
in the same process.  One JSON line per zip is printed and appended to --out.

    python tools/measure_unzip.py [--out results/h100_unzip.jsonl] [--trees numpy_scipy,torch_lib,small_files] [--reps 1]
"""
import argparse
import filecmp
import json
import os
import shutil
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
from measure_zip import SITE, best, make_tree  # noqa: E402


def tree_root(name, tmp):
    if name == "torch_lib":
        root = os.path.join(tmp, name)
        shutil.copytree(os.path.join(SITE, "torch", "lib"), os.path.join(root, "lib"), symlinks=True)
        return root
    return make_tree(name, tmp)


def same_tree(a, b):
    for dirpath, dirnames, filenames in os.walk(a):
        rel = os.path.relpath(dirpath, a)
        other = os.path.join(b, rel)
        if sorted(dirnames) != sorted(d for d in os.listdir(other) if os.path.isdir(os.path.join(other, d))):
            return False
        files = sorted(f for f in os.listdir(other) if not os.path.isdir(os.path.join(other, f)))
        if sorted(filenames) != files:
            return False
        _, mismatch, errors = filecmp.cmpfiles(dirpath, other, filenames, shallow=False)
        if mismatch or errors:
            return False
    return True


def measure(ctx, tree, writer, zip_path, tmp, gpu, reps):
    out_gpu, out_ref = os.path.join(tmp, "x_gpu"), os.path.join(tmp, "x_ref")

    def fresh(d):
        shutil.rmtree(d, ignore_errors=True)
        return d

    def gpu_extract():
        return zipfile_gpu.extract_zip(zip_path, fresh(out_gpu), ctx=ctx)

    def ref_extract():
        with zipfile.ZipFile(zip_path) as zf:
            zf.extractall(fresh(out_ref))

    def ref_test():
        with zipfile.ZipFile(zip_path) as zf:
            return zf.testzip()

    gpu_s, st = best(gpu_extract, reps)
    ref_s, _ = best(ref_extract, reps)
    tgpu_s, bad_gpu = best(lambda: zipfile_gpu.testzip(zip_path, ctx=ctx), reps)
    tref_s, bad_ref = best(ref_test, reps)
    t0 = time.perf_counter()
    identical = same_tree(out_ref, out_gpu) and same_tree(out_gpu, out_ref)
    cmp_s = time.perf_counter() - t0
    shutil.rmtree(out_gpu, ignore_errors=True)
    shutil.rmtree(out_ref, ignore_errors=True)
    kernel_ms = st["kernel_ms"]
    return {
        "tree": tree, "zip_writer": writer, "gpu": gpu, "members": st["members"], "gpu_members": st["gpu_members"],
        "stdlib_members": st["stdlib_members"], "zip_bytes": os.path.getsize(zip_path), "out_bytes": st["out_bytes"],
        "batches": st["batches"], "n_stored": st["n_stored"], "n_small": st["n_small"], "n_large": st["n_large"],
        "n_spans": st["n_spans"], "n_rounds": st["n_rounds"], "n_rejected": st["n_rejected"],
        "copy_ms": round(st["copy_ms"], 3), "small_ms": round(st["small_ms"], 3), "find_ms": round(st["find_ms"], 3),
        "count_ms": round(st["count_ms"], 3), "decode_ms": round(st["decode_ms"], 3),
        "resolve_ms": round(st["resolve_ms"], 3), "crc_ms": round(st["crc_ms"], 3), "h2d_ms": round(st["h2d_ms"], 3),
        "kernel_ms": round(kernel_ms, 3), "kernel_GBps_out": round(st["out_bytes"] / (kernel_ms / 1e3) / 1e9, 3) if kernel_ms else None,
        "e2e_extract_zip_s": round(gpu_s, 3), "e2e_extractall_s": round(ref_s, 3), "extract_speedup": round(ref_s / gpu_s, 2),
        "e2e_testzip_gpu_s": round(tgpu_s, 3), "e2e_testzip_stdlib_s": round(tref_s, 3),
        "testzip_speedup": round(tref_s / tgpu_s, 2), "testzip_gpu": bad_gpu, "testzip_stdlib": bad_ref,
        "trees_identical": identical, "compare_s": round(cmp_s, 2), "reps": reps,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_unzip.jsonl"))
    ap.add_argument("--trees", default="numpy_scipy,torch_lib,small_files")
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:
        tmp = tempfile.mkdtemp(prefix="lb2_unzip_")
        try:
            warm = os.path.join(tmp, "warm")
            os.makedirs(warm)
            with open(os.path.join(warm, "w.bin"), "wb") as f:
                f.write(os.urandom(1 << 20) + bytes(4 << 20))
            zipfile_gpu.zip_tree(warm, os.path.join(tmp, "warm.zip"), ctx=ctx)
            zipfile_gpu.extract_zip(os.path.join(tmp, "warm.zip"), os.path.join(tmp, "warm_x"), ctx=ctx)  # module load
            for name in args.trees.split(","):
                root = tree_root(name, tmp)
                zips = {"make_archive": shutil.make_archive(os.path.join(tmp, name + "_ref"), "zip", root),
                        "zip_tree": os.path.join(tmp, name + "_gpu.zip")}
                zipfile_gpu.zip_tree(root, zips["zip_tree"], ctx=ctx)
                shutil.rmtree(root)
                for writer, path in zips.items():
                    line = json.dumps(measure(ctx, name, writer, path, tmp, gpu, args.reps))
                    print(line, flush=True)
                    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                    with open(args.out, "a") as f:
                        f.write(line + "\n")
                    os.remove(path)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
