"""zip_build (wheels to a Lambda zip: pip's target install and the clean-up restated, shared objects inflated,
stripped and deflated on the GPU) against the literal passes.

Workloads: the installed numpy and scipy as two wheels ("numpy_scipy_wheels"), and the installed torch re-packed as
one wheel ("torch_wheel").  Each wheel holds the files its distribution's RECORD lists, zlib level 6.  For every
workload, end to end on the same disk, with the CUDA context created before any clock starts:
  - the literal passes, each timed: `pip install --no-deps --no-index --target build W...`, the build script's
    clean-up lines, `find -name "*.so" | xargs strip`, shutil.make_archive (zlib level 6);
  - zip_build, without and with a seek table in the zip ("_zst").
No existing GPU composition installs a wheel, so there is no third column.  The zips are compared with
make_archive's: the same names and every file entry's bytes ("trees_identical").  Zip sizes, the bytes that crossed
the bus, the bytes copied against the bytes deflated, the kernel times per engine (CUDA events), the card name and
its power limit are read in the same process.  One JSON line per workload is printed and appended to --out.

    python tools/measure_zip_build.py [--out results/h100_zip_build.jsonl] [--cases numpy_scipy_wheels,torch_wheel]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import layer  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402
from measure_zip_tarballs import same_files, sm_clock  # noqa: E402
from test_gpu_layer_build import installed_wheel  # noqa: E402
from test_layer_build_host import cleanup_lines, pip_install  # noqa: E402

CASES = {"numpy_scipy_wheels": ["numpy", "scipy"], "torch_wheel": ["torch"]}


def literal_passes(wheels, tmp, prefix):
    """pip --target, the clean-up lines, the strip line, make_archive; (zip, seconds of each pass)"""
    work = os.path.join(tmp, "work")
    build = os.path.join(work, "build")
    t0 = time.perf_counter()
    pip_install(build, wheels)
    t1 = time.perf_counter()
    cleanup_lines(work, ())
    t2 = time.perf_counter()
    subprocess.run('find %s/ -name "*.so" | xargs strip' % build, shell=True)
    t3 = time.perf_counter()
    tree = os.path.join(tmp, "tree")
    os.makedirs(tree)
    os.rename(build, os.path.join(tree, prefix[:-1]))
    t4 = time.perf_counter()
    out = shutil.make_archive(os.path.join(tmp, "passes"), "zip", tree)
    t5 = time.perf_counter()
    shutil.rmtree(tree)
    shutil.rmtree(work)
    return out, (t1 - t0, t2 - t1, t3 - t2, t5 - t4)


def measure(ctx, case, wheels, tmp, gpu, prefix="python/"):
    out = {"case": case, "gpu": gpu, "sm_clock": sm_clock(), "wheels": len(wheels),
           "src_bytes": sum(os.path.getsize(w) for w in wheels)}
    t0 = time.perf_counter()
    ref, passes = literal_passes(wheels, tmp, prefix)
    ref_s = time.perf_counter() - t0
    out.update({"e2e_literal_passes_s": round(ref_s, 3), "pip_target_s": round(passes[0], 3),
                "cleanup_s": round(passes[1], 3), "find_xargs_strip_s": round(passes[2], 3),
                "make_archive_s": round(passes[3], 3), "make_archive_bytes": os.path.getsize(ref)})
    for tag, kw in (("", {}), ("_zst", {"seek_table": True})):
        dst = os.path.join(tmp, "layer.zip")
        t0 = time.perf_counter()
        st = layer.zip_build(dst, (), wheels, prefix=prefix, ctx=ctx, **kw)
        s = time.perf_counter() - t0
        out.update({"e2e_zip_build%s_s" % tag: round(s, 3), "speedup_vs_passes%s" % tag: round(ref_s / s, 2),
                    "zip_bytes%s" % tag: st["zip_bytes"], "kernel_ms%s" % tag: round(st["kernel_ms"], 3),
                    "trees_identical%s" % tag: same_files(ref, dst)})
        if not tag:
            un, sp, df = st["unzip"], st["strip"], st["deflate"]
            out.update({
                "wheel_members": st["wheel_members"], "entries": st["entries"], "selected": st["selected"],
                "gpu_members": st["gpu"], "fallback": st["fallback"], "skipped": st["skipped"],
                "removed_entries": st["removed"]["entries"], "generated_scripts": st["generated_scripts"],
                "so_bytes_in": st["in_bytes"], "so_bytes_out": st["out_bytes"],
                "copied_members": st["copied"]["members"], "copied_bytes": st["copied"]["bytes"],
                "deflated_file_bytes": st["file_bytes"], "deflated_bytes": st["deflated_bytes"],
                "uploaded_bytes": st["uploaded_bytes"], "downloaded_bytes": st["downloaded_bytes"],
                "inflate_kernel_ms": round(un["kernel_ms"], 3), "plan_ms": round(sp["plan_ms"], 3),
                "compact_ms": round(sp["compact_ms"], 3), "strip_kernel_ms": round(sp["plan_ms"] + sp["compact_ms"], 3),
                "deflate_kernel_ms": round(df["kernel_ms"], 3), "gather_ms": round(df["h2d_ms"], 3),
            })
        os.remove(dst)
    os.remove(ref)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_zip_build.jsonl"))
    ap.add_argument("--cases", default="numpy_scipy_wheels,torch_wheel")
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:   # no device: this raises, nothing is timed
        tmp = tempfile.mkdtemp(prefix="lb2_zip_build_")
        try:
            wdir = os.path.join(tmp, "wheels")
            os.makedirs(wdir)
            warm = installed_wheel("numpy", wdir)   # module load and first allocations of every engine
            for level in (None, 9):
                layer.zip_build(os.path.join(tmp, "warm.zip"), (), [warm], ctx=ctx, compresslevel=level)
            os.remove(warm)
            for case in args.cases.split(","):
                wheels = [installed_wheel(d, wdir) for d in CASES[case]]
                line = json.dumps(measure(ctx, case, wheels, tmp, gpu))
                print(line, flush=True)
                os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                with open(args.out, "a") as f:
                    f.write(line + "\n")
                for w in wheels:
                    os.remove(w)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
