"""check_zip(symbols=True) (the symbol lookups of a zip's shared objects on the GPU) against check_zip without it and
against the host route on the same machine: `ZipFile.extractall`, then the loader's own trace with every binding
done (`LD_TRACE_LOADED_OBJECTS=1 LD_WARN=yes LD_BIND_NOW=yes ld.so --library-path P ROOT`) per root checked.

Workloads: numpy + scipy as a layer zip written by shutil.make_archive ("numpy_scipy_make_archive") and by zip_tree
with seek tables ("numpy_scipy_zip_tree_seek"), and torch/lib zipped by make_archive ("torch_lib"); the same zips as
tools/measure_deps.py.  The runtime libraries are the host's (/lib/x86_64-linux-gnu) and the interpreter is
sys.executable, so every lookup runs.  Recorded per workload: references, lookups, the index / references / resolve
kernel times and their sum (CUDA events), the bytes up and down with and without symbols, check_zip end to end with
and without symbols (after one warm-up of each), the inflate kernel time, and the host route, with the card name and
its power limit read in the same process.  The CUDA context exists before any clock starts.  One JSON line per
workload is printed and appended to --out.

    python tools/measure_symbols.py [--out results/h100_symbols.jsonl] [--cases numpy_scipy_make_archive,torch_lib]
"""
import argparse
import json
import os
import posixpath
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
from measure_deps import make_zip  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402

CASES = ("numpy_scipy_make_archive", "numpy_scipy_zip_tree_seek", "torch_lib")
HOST_LIBS = "/lib/x86_64-linux-gnu"
LD_SO = "/lib64/ld-linux-x86-64.so.2"


def host_route(zip_path, mount, roots, tmp):
    t0 = time.perf_counter()
    d = os.path.join(tmp, "x")
    with zipfile.ZipFile(zip_path) as zf:
        zf.extractall(d + mount)
    t1 = time.perf_counter()
    env = dict(os.environ, LD_TRACE_LOADED_OBJECTS="1", LD_WARN="yes", LD_BIND_NOW="yes")
    for r in roots:
        subprocess.run([LD_SO, "--library-path", d + posixpath.dirname(r), d + r], env=env, stdout=subprocess.DEVNULL,
                       stderr=subprocess.DEVNULL)
    t2 = time.perf_counter()
    shutil.rmtree(d)
    return t1 - t0, t2 - t1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_symbols.jsonl"))
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    info = gpu_info()
    kw = {"symbols": True, "interpreter": [sys.executable], "runtime_libs": [HOST_LIBS]}
    with N.Context(0) as ctx, tempfile.TemporaryDirectory() as tmp:
        for case in args.cases.split(","):
            zip_path, mount = make_zip(case, tmp, ctx)
            deps.check_zip(zip_path, mount=mount, ctx=ctx)  # warm-up of each form
            deps.check_zip(zip_path, mount=mount, ctx=ctx, **kw)
            t0 = time.perf_counter()
            plain = deps.check_zip(zip_path, mount=mount, ctx=ctx)
            t1 = time.perf_counter()
            rep = deps.check_zip(zip_path, mount=mount, ctx=ctx, **kw)
            t2 = time.perf_counter()
            checked = [r for r in rep["closures"] if not any(x["how"] == "missing" for x in rep["resolved"][r])]
            extract_s, trace_s = host_route(zip_path, mount, checked, tmp)
            st, ps = rep["stats"], plain["stats"]
            row = {"case": case, "zip_bytes": os.path.getsize(zip_path), "roots": st["roots"], "objects": st["objects"],
                   "roots_checked": len(checked), "symbols_skipped": st["symbols_skipped"],
                   "references": st["references"], "lookups": st["lookups"],
                   "symbols_ms": round(st["symbols_ms"], 3), "index_ms": round(st["symbols_index_ms"], 3),
                   "refs_ms": round(st["symbols_refs_ms"], 3), "resolve_ms": round(st["symbols_resolve_ms"], 3),
                   "inflate_ms": round(st["inflate_ms"], 3), "parse_ms": round(st["parse_ms"], 3),
                   "bytes_up": st["bytes_up"], "bytes_down": st["bytes_down"],
                   "bytes_up_without_symbols": ps["bytes_up"], "bytes_down_without_symbols": ps["bytes_down"],
                   "check_zip_symbols_s": round(t2 - t1, 3), "check_zip_s": round(t1 - t0, 3),
                   "host_extractall_s": round(extract_s, 3), "host_ld_trace_s": round(trace_s, 3),
                   "host_total_s": round(extract_s + trace_s, 3),
                   "problems": len(rep["problems"]), "symbol_problems": sum(p["kind"] == "symbol" for p in rep["problems"]),
                   "gpu": info}
            print(json.dumps(row))
            with open(args.out, "a") as f:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
