"""zip_tarballs (package tarballs to a Lambda zip, inflated, stripped and deflated on the GPU) against two baselines.

Cases: numpy + numpy.libs and scipy + scipy.libs as two assets ("numpy_scipy_two"), all four as one asset
("numpy_scipy_one"), and torch/lib ("torch_lib").  Each asset is written by tarfile "w:gz" (zlib level 9, no seek
table), by gzip_tarball and by gzip_tarball(seek_table=True).  For every case and writer, end to end on the same
disk, with the CUDA context created before any clock starts:
  - the four literal passes: tarfile "r:gz" extractall of each asset, the reference's `find -name "*.so" | xargs
    strip`, shutil.make_archive (zlib level 6);
  - the existing GPU composition: extract_tarball of each asset, strip_tree, zip_tree;
  - zip_tarballs at the default level, without and with a seek table in the zip ("_zst"), and, for the cases in
    --l9, at --level 9 ("_l9").
The zips are compared with make_archive's: the same names, and every file entry's bytes ("trees_identical").  Zip
sizes, the bytes that crossed the bus, the kernel times per engine (CUDA events), the card name, its power limit and
its SM clock are read in the same process.  One JSON line per (case, writer) is printed and appended to --out.

    python tools/measure_zip_tarballs.py [--out results/h100_zip_tarballs.jsonl]
                                         [--cases numpy_scipy_two,numpy_scipy_one,torch_lib]
                                         [--writers tarfile,gzip_tarball,gzip_tarball_seek] [--l9 numpy_scipy_two]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tarfile
import tempfile
import time
import zipfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import layer, strip, tarball, zipfile_gpu  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402
from measure_zip import SITE  # noqa: E402

CASES = {
    "numpy_scipy_two": [["numpy", "numpy.libs"], ["scipy", "scipy.libs"]],
    "numpy_scipy_one": [["numpy", "numpy.libs", "scipy", "scipy.libs"]],
    "torch_lib": [["torch/lib"]],
}


def sm_clock():
    r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown"


def write_assets(ctx, case, writer, tmp):
    srcs = []
    for k, dirs in enumerate(CASES[case]):
        paths = [os.path.join(SITE, d) for d in dirs if os.path.exists(os.path.join(SITE, d))]
        if not paths:
            raise RuntimeError("%s: none of %s is installed" % (case, dirs))
        src = os.path.join(tmp, "%s_%d_%s.tar.gz" % (case, k, writer))
        if writer == "tarfile":
            with tarfile.open(src, "w:gz") as tar:
                for p in paths:
                    tar.add(p, arcname=os.path.basename(p))
        else:
            tarball.gzip_tarball(paths, src, ctx=ctx, seek_table=writer == "gzip_tarball_seek")
        srcs.append(src)
    return srcs


def four_passes(srcs, tmp, prefix):
    """tarfile extractall of each source, the strip line, make_archive; (zip, seconds of each pass)"""
    d = os.path.join(tmp, "passes")
    t0 = time.perf_counter()
    for s in srcs:
        with tarfile.open(s, "r:gz") as tar:
            tar.extractall(os.path.join(d, prefix), filter="fully_trusted")
    t1 = time.perf_counter()
    subprocess.run('find %s/ -name "*.so" | xargs strip' % d, shell=True)
    t2 = time.perf_counter()
    out = shutil.make_archive(os.path.join(tmp, "passes"), "zip", d)
    t3 = time.perf_counter()
    shutil.rmtree(d)
    return out, (t1 - t0, t2 - t1, t3 - t2)


def gpu_composition(ctx, srcs, tmp, prefix):
    """extract_tarball of each source, strip_tree, zip_tree; (zip, seconds of each step)"""
    d = os.path.join(tmp, "composed")
    t0 = time.perf_counter()
    for s in srcs:
        tarball.extract_tarball(s, os.path.join(d, prefix), ctx=ctx)
    t1 = time.perf_counter()
    strip.strip_tree(d, ctx=ctx)
    t2 = time.perf_counter()
    out = os.path.join(tmp, "composed.zip")
    zipfile_gpu.zip_tree(d, out, ctx=ctx)
    t3 = time.perf_counter()
    shutil.rmtree(d)
    return out, (t1 - t0, t2 - t1, t3 - t2)


def same_files(a_path, b_path):
    with zipfile.ZipFile(a_path) as a, zipfile.ZipFile(b_path) as b:
        if sorted(a.namelist()) != sorted(b.namelist()):
            return False
        return all(zi.is_dir() or a.read(zi) == b.read(zi.filename) for zi in a.infolist())


def measure(ctx, case, writer, srcs, tmp, gpu, level9, prefix="python/"):
    out = {"case": case, "writer": writer, "gpu": gpu, "sm_clock": sm_clock(), "sources": len(srcs),
           "src_bytes": sum(os.path.getsize(s) for s in srcs)}
    t0 = time.perf_counter()
    ref, passes = four_passes(srcs, tmp, prefix)
    ref_s = time.perf_counter() - t0
    out.update({"e2e_four_passes_s": round(ref_s, 3), "extract_s": round(passes[0], 3),
                "find_xargs_strip_s": round(passes[1], 3), "make_archive_s": round(passes[2], 3),
                "make_archive_bytes": os.path.getsize(ref)})
    t0 = time.perf_counter()
    comp, steps = gpu_composition(ctx, srcs, tmp, prefix)
    comp_s = time.perf_counter() - t0
    out.update({"e2e_gpu_composition_s": round(comp_s, 3), "extract_tarball_s": round(steps[0], 3),
                "strip_tree_s": round(steps[1], 3), "zip_tree_s": round(steps[2], 3),
                "gpu_composition_bytes": os.path.getsize(comp), "gpu_composition_identical": same_files(ref, comp)})
    os.remove(comp)
    runs = [("", {}), ("_zst", {"seek_table": True})] + ([("_l9", {"compresslevel": 9})] if level9 else [])
    for tag, kw in runs:
        dst = os.path.join(tmp, "layer.zip")
        t0 = time.perf_counter()
        st = layer.zip_tarballs(srcs, dst, prefix=prefix, ctx=ctx, **kw)
        s = time.perf_counter() - t0
        out.update({"e2e_zip_tarballs%s_s" % tag: round(s, 3), "speedup_vs_passes%s" % tag: round(ref_s / s, 2),
                    "speedup_vs_composition%s" % tag: round(comp_s / s, 2), "zip_bytes%s" % tag: st["zip_bytes"],
                    "kernel_ms%s" % tag: round(st["kernel_ms"], 3),
                    "deflate_ms%s" % tag: round(st["deflate"]["kernel_ms"], 3),
                    "trees_identical%s" % tag: same_files(ref, dst)})
        if not tag:
            inf, ix, sp, df = st["inflate"], st["index"], st["strip"], st["deflate"]
            out.update({
                "members": st["members"], "entries": st["entries"],
                "selected": st["selected"], "gpu_members": st["gpu"], "fallback": st["fallback"],
                "skipped": st["skipped"], "so_bytes_in": st["in_bytes"], "so_bytes_out": st["out_bytes"],
                "tar_bytes_in": st["tar_bytes_in"], "uploaded_bytes": st["uploaded_bytes"],
                "downloaded_bytes": st["downloaded_bytes"], "inflate_kernel_ms": round(inf["kernel_ms"], 3),
                "inflate_seek_table": inf.get("seek_table", 0), "index_ms": round(ix["kernel_ms"], 3),
                "index_misses": ix["misses"], "plan_ms": round(sp["plan_ms"], 3),
                "compact_ms": round(sp["compact_ms"], 3), "gather_ms": round(df["h2d_ms"], 3),
            })
        os.remove(dst)
    os.remove(ref)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_zip_tarballs.jsonl"))
    ap.add_argument("--cases", default="numpy_scipy_two,numpy_scipy_one,torch_lib")
    ap.add_argument("--writers", default="tarfile,gzip_tarball,gzip_tarball_seek")
    ap.add_argument("--l9", default="numpy_scipy_two", help="cases also measured at --level 9")
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:   # no device: this raises, nothing is timed
        tmp = tempfile.mkdtemp(prefix="lb2_zip_tarballs_")
        try:
            warm = os.path.join(tmp, "warm.tar.gz")   # module load and first allocations of every engine
            with tarfile.open(warm, "w:gz") as tar:
                tar.add(os.path.join(ROOT, "tests", "golden", "cxx_g.in.bin"), "warm/cxx_g.so")
            for level in (None, 9):
                layer.zip_tarballs([warm, warm], os.path.join(tmp, "warm.zip"), ctx=ctx, compresslevel=level)
            gpu_composition(ctx, [warm], tmp, "")
            for case in args.cases.split(","):
                for writer in args.writers.split(","):
                    srcs = write_assets(ctx, case, writer, tmp)
                    line = json.dumps(measure(ctx, case, writer, srcs, tmp, gpu, case in args.l9.split(",")))
                    print(line, flush=True)
                    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                    with open(args.out, "a") as f:
                        f.write(line + "\n")
                    for s in srcs:
                        os.remove(s)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
