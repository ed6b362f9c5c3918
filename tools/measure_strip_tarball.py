"""strip_tarball (inflate, strip and deflate chained on the GPU) against the three passes it replaces.

For each tree -- numpy + numpy.libs + scipy + scipy.libs and torch/lib -- the tree is tarred twice: by tarfile "w:gz"
(zlib level 9 in one stream, no flush points, what the reference's create_compressed_tarball writes) and by
gzip_tarball (the GPU writer).  Each tarball is then stripped, end to end:
  - by tarball.strip_tarball at the default level and at --level 9, on a context created before the clock starts;
  - by tarfile "r:gz" extractall, the reference's `find -name "*.so" | xargs strip` and tarfile "w:gz", on the same
    disk.
The results are compared member by member (the same names in the same order, every regular member's bytes).  Asset
sizes, the bytes that crossed the bus, the inflate, index, strip, gather and deflate kernel times (CUDA events), the
card name and its power limit are read in the same process.  One JSON line per (tree, writer) is printed and
appended to --out.

    python tools/measure_strip_tarball.py [--out results/h100_strip_tarball.jsonl] [--trees numpy_scipy,torch_lib]
                                          [--writers tarfile,gzip_tarball]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import tarball  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402
from measure_unzip import tree_root  # noqa: E402
from measure_zip import best  # noqa: E402


def three_passes(src, tmp):
    """tarfile "r:gz" extractall + the reference's strip line + tarfile "w:gz"; (the tarball, seconds of each pass)"""
    d = os.path.join(tmp, "passes")
    shutil.rmtree(d, ignore_errors=True)
    t0 = time.perf_counter()
    with tarfile.open(src, "r:gz") as tar:
        tar.extractall(d, filter="fully_trusted")
    t1 = time.perf_counter()
    rc = subprocess.run('find %s/ -name "*.so" | xargs strip' % d, shell=True).returncode
    t2 = time.perf_counter()
    out = os.path.join(tmp, "passes_out.tar.gz")
    with tarfile.open(out, "w:gz") as tar:
        for name in sorted(os.listdir(d)):
            tar.add(os.path.join(d, name), arcname=name)
    t3 = time.perf_counter()
    shutil.rmtree(d)
    if rc:
        raise RuntimeError("the reference's strip line exited %d" % rc)
    return out, (t1 - t0, t2 - t1, t3 - t2)


def same_members(a_path, b_path):
    with tarfile.open(a_path, "r:gz") as a, tarfile.open(b_path, "r:gz") as b:
        ma, mb = a.getmembers(), b.getmembers()
        if [m.name for m in ma] != [m.name for m in mb]:
            return False
        for x, y in zip(ma, mb):
            if x.type != y.type or x.linkname != y.linkname:
                return False
            if x.isreg() and a.extractfile(x).read() != b.extractfile(y).read():
                return False
    return True


def measure(ctx, name, writer, src, tmp, gpu):
    out = {"tree": name, "writer": writer, "gpu": gpu, "src_bytes": os.path.getsize(src)}
    ref_s, (ref_tgz, passes) = best(lambda: three_passes(src, tmp), 1)
    out.update({"e2e_three_passes_s": round(ref_s, 3), "extract_s": round(passes[0], 3),
                "find_xargs_strip_s": round(passes[1], 3), "write_gz_s": round(passes[2], 3),
                "three_pass_bytes": os.path.getsize(ref_tgz)})
    for level in (None, 9):
        dst = os.path.join(tmp, "%s_%s_stripped.tar.gz" % (name, writer))
        gpu_s, st = best(lambda: tarball.strip_tarball(src, dst, ctx=ctx, compresslevel=level), 1)
        tag = "" if level is None else "_l9"
        inf, ix, sp, df = st["inflate"], st["index"], st["strip"], st["deflate"]
        out.update({
            "e2e_strip_tarball%s_s" % tag: round(gpu_s, 3), "speedup%s" % tag: round(ref_s / gpu_s, 2),
            "dst_bytes%s" % tag: st["dst_bytes"], "deflate_ms%s" % tag: round(df["deflate_ms"] + df["crc_ms"], 3),
            "kernel_ms%s" % tag: round(st["kernel_ms"], 3), "members_identical%s" % tag: same_members(ref_tgz, dst),
        })
        if level is None:
            out.update({
                "members": st["members"], "selected": st["selected"], "gpu_members": st["gpu"],
                "fallback": st["fallback"], "skipped": st["skipped"], "so_bytes_in": st["in_bytes"],
                "so_bytes_out": st["out_bytes"], "tar_bytes_in": st["tar_bytes_in"], "tar_bytes_out": st["tar_bytes_out"],
                "uploaded_bytes": st["uploaded_bytes"], "downloaded_bytes": st["downloaded_bytes"],
                "inflate_kernel_ms": round(inf["kernel_ms"], 3), "index_ms": round(ix["kernel_ms"], 3),
                "index_members": ix["n_members"], "index_misses": ix["misses"], "plan_ms": round(sp["plan_ms"], 3),
                "compact_ms": round(sp["compact_ms"], 3), "gather_ms": round(df["h2d_ms"], 3),
            })
        os.remove(dst)
    os.remove(ref_tgz)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_strip_tarball.jsonl"))
    ap.add_argument("--trees", default="numpy_scipy,torch_lib")
    ap.add_argument("--writers", default="tarfile,gzip_tarball")
    args = ap.parse_args()
    gpu = gpu_info()
    with N.Context(0) as ctx:   # no device: this raises, nothing is timed
        tmp = tempfile.mkdtemp(prefix="lb2_strip_tarball_")
        try:
            warm = os.path.join(tmp, "warm.tar.gz")   # module load and first allocations of the engines
            with tarfile.open(warm, "w:gz") as tar:
                tar.add(os.path.join(ROOT, "tests", "golden", "cxx_g.in.bin"), "warm/cxx_g.so")
            for level in (None, 9):
                tarball.strip_tarball(warm, os.path.join(tmp, "warm_out.tar.gz"), ctx=ctx, compresslevel=level)
            for name in args.trees.split(","):
                root = tree_root(name, tmp)
                for writer in args.writers.split(","):
                    src = os.path.join(tmp, "%s_%s.tar.gz" % (name, writer))
                    if writer == "tarfile":
                        with tarfile.open(src, "w:gz") as tar:
                            for entry in sorted(os.listdir(root)):
                                tar.add(os.path.join(root, entry), arcname=entry)
                    else:
                        tarball.gzip_tarball([os.path.join(root, e) for e in sorted(os.listdir(root))], src, ctx=ctx)
                    line = json.dumps(measure(ctx, name, writer, src, tmp, gpu))
                    print(line, flush=True)
                    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                    with open(args.out, "a") as f:
                        f.write(line + "\n")
                    os.remove(src)
                shutil.rmtree(root)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
