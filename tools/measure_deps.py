"""check_zip (the dynamic sections of a zip's shared objects read on the GPU, the loader's search restated on the host)
against the host route on the same machine: `ZipFile.extractall`, then `readelf -dVW` on every object check_zip
parsed (the resolver is the same code on both routes and is not timed on the host route).

Workloads: numpy + scipy as a layer zip (prefix python/, mount /opt) written by shutil.make_archive
("numpy_scipy_make_archive") and by zip_tree with seek tables ("numpy_scipy_zip_tree_seek"), and torch/lib zipped by
make_archive ("torch_lib", mount /opt/python/torch).  Recorded per workload: objects parsed, rounds, bytes up and
down, the inflate and parse kernel times (CUDA events), check_zip end to end and the host route, with the card name
and its power limit read in the same process.  The CUDA context exists before any clock starts.  One JSON line per
workload is printed and appended to --out.

    python tools/measure_deps.py [--out results/h100_deps.jsonl] [--cases numpy_scipy_make_archive,torch_lib]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import deps  # noqa: E402
from lambdipy_b200 import zipfile_gpu as Z  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402
import elf_fixtures as F  # noqa: E402

CASES = ("numpy_scipy_make_archive", "numpy_scipy_zip_tree_seek", "torch_lib")


def make_zip(case, tmp, ctx):
    """(zip path, mount)"""
    sp = F.site_packages()
    if case == "torch_lib":
        return shutil.make_archive(os.path.join(tmp, "torch_lib"), "zip", os.path.join(sp, "torch"), "lib"), \
            "/opt/python/torch"
    tree = os.path.join(tmp, "tree")
    if not os.path.isdir(tree):
        for r in ("numpy", "scipy", "numpy.libs", "scipy.libs"):
            shutil.copytree(os.path.join(sp, r), os.path.join(tree, "python", r), symlinks=True,
                            ignore=shutil.ignore_patterns("__pycache__"))
    if case == "numpy_scipy_make_archive":
        return shutil.make_archive(os.path.join(tmp, "ma"), "zip", tree), "/opt"
    out = os.path.join(tmp, "zt.zip")
    Z.zip_tree(tree, out, ctx=ctx, seek_table=True)
    return out, "/opt"


def host_route(zip_path, members, tmp):
    t0 = time.perf_counter()
    d = os.path.join(tmp, "x")
    with zipfile.ZipFile(zip_path) as zf:
        zf.extractall(d)
    t1 = time.perf_counter()
    for m in members:
        subprocess.run(["readelf", "-dVW", os.path.join(d, m)], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    t2 = time.perf_counter()
    shutil.rmtree(d)
    return t1 - t0, t2 - t1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_deps.jsonl"))
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    info = gpu_info()
    with N.Context(0) as ctx, tempfile.TemporaryDirectory() as tmp:
        for case in args.cases.split(","):
            zip_path, mount = make_zip(case, tmp, ctx)
            deps.check_zip(zip_path, mount=mount, ctx=ctx)  # warm-up: pinned buffers, module load
            t0 = time.perf_counter()
            rep = deps.check_zip(zip_path, mount=mount, ctx=ctx)
            gpu_s = time.perf_counter() - t0
            members = sorted({o["member"] for o in rep["objects"].values()})
            extract_s, readelf_s = host_route(zip_path, members, tmp)
            st = rep["stats"]
            row = {"case": case, "zip_bytes": os.path.getsize(zip_path), "members": st["members"], "roots": st["roots"],
                   "objects": st["objects"], "rounds": st["rounds"], "bytes_up": st["bytes_up"],
                   "bytes_down": st["bytes_down"], "inflate_ms": round(st["inflate_ms"], 3),
                   "parse_ms": round(st["parse_ms"], 3), "check_zip_s": round(gpu_s, 3),
                   "host_extractall_s": round(extract_s, 3), "host_readelf_s": round(readelf_s, 3),
                   "host_total_s": round(extract_s + readelf_s, 3), "problems": len(rep["problems"]),
                   "max_versions": rep["max_versions"], "gpu": info}
            print(json.dumps(row))
            with open(args.out, "a") as f:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
