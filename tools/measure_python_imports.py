"""check_zip(python="3.12") (CPython's import finder restated on the host, each module's PyInit_* looked up on the
GPU by lb2_syms_find) against check_zip without it and against the host route on the same machine: `extractall`,
then importlib's PathFinder with the target's FileFinder loaders for every module name, and `ctypes.CDLL(path,
RTLD_NOW | RTLD_LOCAL)` + `hasattr(lib, "PyInit_...")` for every module it finds.

Workloads: numpy + scipy as a layer zip written by shutil.make_archive and by zip_tree with seek tables (the zips of
tools/measure_deps.py, mount /opt), and torch/lib zipped under python/torch/lib (mount /opt), whose *.so are
libraries the finder reaches by name and which export no PyInit_*.  Per workload, three alternating runs of
check_zip without and with python (after one warm-up of each): the median and the spread of each, the find kernel's
time (CUDA events) and query count, and, from one run with the engines in hand, the index kernels' time that
python=... adds when symbols=False.  The card name and power limit are read in the same process.  One JSON line per
workload is printed and appended to --out.

    python tools/measure_python_imports.py [--out results/h100_python_imports.jsonl] [--cases ...]
"""
import argparse
import json
import os
import shutil
import statistics
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
from measure_deps import make_zip  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402

CASES = ("numpy_scipy_make_archive", "numpy_scipy_zip_tree_seek", "torch_lib")
VERSION = "3.12"


def torch_lib_zip(tmp):
    import elf_fixtures as F
    lib = os.path.join(F.site_packages(), "torch", "lib")
    p = os.path.join(tmp, "torch_lib_py.zip")
    with zipfile.ZipFile(p, "w", zipfile.ZIP_DEFLATED) as zf:
        for name in sorted(os.listdir(lib)):
            f = os.path.join(lib, name)
            if os.path.isfile(f) and not os.path.islink(f):
                zf.write(f, "python/torch/lib/" + name)
    return p, "/opt"


def host_route(zip_path, mount, tmp):
    """(extract s, finder + dlsym s, modules found) of the route without the GPU"""
    import ctypes
    from test_python_imports_host import oracle
    t0 = time.perf_counter()
    root = os.path.join(tmp, "x")
    with zipfile.ZipFile(zip_path) as zf:
        zf.extractall(root + mount)
    t1 = time.perf_counter()
    find = oracle(root, VERSION, "x86_64", mount)
    finder = deps._Finder(deps._Tree([], mount), VERSION, "x86_64")
    found = 0
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)[len(root):]
            got = finder.name(p) if f.endswith(".so") else None
            if got and got[2] is None and find(got[0]) == p:
                try:  # torch/lib's libraries need CUDA libraries the zip does not carry
                    lib = ctypes.CDLL(root + p, os.RTLD_NOW | os.RTLD_LOCAL)
                except OSError:
                    continue
                found += hasattr(lib, deps.export_name(got[0]).decode())
    t2 = time.perf_counter()
    shutil.rmtree(root)
    return t1 - t0, t2 - t1, found


def engines_run(ctx, zip_path, mount):
    """the resolver's stats of one check_zip(python=...) run with the engines in hand"""
    with Z.GpuUnzipDecoder(ctx) as dec, deps.GpuElfParser(ctx) as parser, deps.GpuSymbolResolver(ctx) as r:
        deps.check_with(zip_path, dec, parser, mount=mount, python=VERSION, resolver=r)
        return r.stats()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_python_imports.jsonl"))
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    info = gpu_info()
    with N.Context(0) as ctx, tempfile.TemporaryDirectory() as tmp:
        for case in args.cases.split(","):
            zip_path, mount = torch_lib_zip(tmp) if case == "torch_lib" else make_zip(case, tmp, ctx)
            deps.check_zip(zip_path, mount=mount, ctx=ctx)  # warm-up of each form
            deps.check_zip(zip_path, mount=mount, ctx=ctx, python=VERSION)
            plain_s, py_s, find_ms = [], [], []
            for _ in range(3):
                t0 = time.perf_counter()
                plain = deps.check_zip(zip_path, mount=mount, ctx=ctx)
                t1 = time.perf_counter()
                rep = deps.check_zip(zip_path, mount=mount, ctx=ctx, python=VERSION)
                t2 = time.perf_counter()
                plain_s.append(t1 - t0)
                py_s.append(t2 - t1)
                find_ms.append(rep["stats"]["find_ms"])
            rs = engines_run(ctx, zip_path, mount)
            extract_s, walk_s, host_found = host_route(zip_path, mount, tmp)
            st, ps = rep["stats"], plain["stats"]
            mods = rep["python"]["modules"].values()
            row = {"case": case, "python": VERSION, "zip_bytes": os.path.getsize(zip_path), "roots": st["roots"],
                   "objects": st["objects"], "modules": st["modules"], "python_skipped": st["python_skipped"],
                   "libraries": sum(m["class"] == "library" for m in mods),
                   "find_queries": st["find_queries"], "find_ms_runs": [round(x, 4) for x in find_ms],
                   "index_ms_added": round(rs["index_ms"] + rs["refs_ms"], 3),
                   "check_zip_s_runs": [round(x, 3) for x in plain_s],
                   "check_zip_python_s_runs": [round(x, 3) for x in py_s],
                   "check_zip_s": round(statistics.median(plain_s), 3),
                   "check_zip_python_s": round(statistics.median(py_s), 3),
                   "bytes_up": st["bytes_up"], "bytes_down": st["bytes_down"],
                   "bytes_up_without_python": ps["bytes_up"], "bytes_down_without_python": ps["bytes_down"],
                   "host_extractall_s": round(extract_s, 3), "host_finder_dlsym_s": round(walk_s, 3),
                   "host_total_s": round(extract_s + walk_s, 3), "host_modules_exporting": host_found,
                   "python_problems": sum(p["kind"] == "python" for p in rep["problems"]), "gpu": info}
            print(json.dumps(row))
            with open(args.out, "a") as f:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
