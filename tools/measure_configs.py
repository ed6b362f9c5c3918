#!/usr/bin/env python
"""Measures BASELINE.json configs 1-3 (real build trees of the installed packages) on a GPU machine and
prints one JSON document: for each tree the reference's own line on host cores (serial, and -P nproc), the
CUDA path device-resident (plan / compaction kernel times, roofline fraction), through host buffers
(lb2_strip_host) and through the in-place tree API (lb2_strip_tree) -- plus a byte-for-byte check of
the GPU-stripped tree against the reference-stripped tree.

    python tools/measure_configs.py > gpurun_out/configs.json
"""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import elf_fixtures as F  # noqa: E402
from bench import peaks  # noqa: E402  (the HBM copy rate of this GPU, measured the way bench.py measures it)
from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import strip as S  # noqa: E402
from lambdipy_b200.device import DeviceBatch  # noqa: E402

TREES = {
    "config1_numpy (stand-in for `lambdipy build numpy==1.17`)": ["numpy", "numpy.libs"],
    "config2_numpy+scipy+sklearn+PIL": ["numpy", "scipy", "sklearn", "PIL", "numpy.libs", "scipy.libs", "pillow.libs", "scikit_learn.libs"],
    "config3_torch (stand-in for tensorflow 1.13.1)": ["torch"],
}
REF = 'find {d}/ -name "*.so" | xargs strip'
PAR = 'find {d}/ -name "*.so" | xargs -P {p} -n 1 strip'


def copy_tree(roots, dst):
    sp = F.site_packages()
    for r in roots:
        shutil.copytree(os.path.join(sp, r), os.path.join(dst, r), symlinks=True,
                        ignore=lambda d, names: [n for n in names if not (os.path.isdir(os.path.join(d, n)) or ".so" in n)])


def selected(root):
    out = []
    for d, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(d, f)
            if f.endswith(".so") and os.path.isfile(p) and not os.path.islink(p):
                out.append(p)
    return sorted(out)


def snapshot(root):
    out = {}
    for p in selected(root):
        with open(p, "rb") as fh:
            out[os.path.relpath(p, root)] = fh.read()
    return out


def best(fn, reps):
    ts = []
    for _ in range(reps):
        ts.append(fn())
    return min(ts), ts


def main():
    nproc = os.cpu_count()
    base = tempfile.mkdtemp(prefix="lb2_cfg_", dir="/dev/shm")
    ctx = N.Context(0)
    peak, peak_src = peaks()
    res = {"nproc": nproc, "strip": subprocess.run(["strip", "--version"], capture_output=True, text=True).stdout.splitlines()[0],
           "hbm_copy_gbs": peak, "hbm_copy_source": peak_src, "trees": {}}
    try:
        for name, roots in TREES.items():
            master = os.path.join(base, "master")
            shutil.rmtree(master, ignore_errors=True)
            os.makedirs(master)
            copy_tree(roots, master)
            files = selected(master)
            in_bytes = sum(os.path.getsize(p) for p in files)
            r = {"files": len(files), "in_bytes": in_bytes}

            def cpu(line):
                run = os.path.join(base, "run")
                shutil.rmtree(run, ignore_errors=True)
                shutil.copytree(master, run, symlinks=True)
                t0 = time.perf_counter()
                rc = subprocess.run(["bash", "-c", "set -o pipefail; " + line.format(d=run, p=nproc)], capture_output=True)
                dt = time.perf_counter() - t0
                assert rc.returncode == 0, rc.stderr[:300]
                return dt

            ser, _ = best(lambda: cpu(REF), 2 if in_bytes > (1 << 30) else 3)
            par, _ = best(lambda: cpu(PAR), 3)
            ref_snap = snapshot(os.path.join(base, "run"))
            r["out_bytes"] = sum(len(v) for v in ref_snap.values())
            r["cpu_serial_s"], r["cpu_serial_gbs"] = ser, in_bytes / 1e9 / ser
            r["cpu_parallel_s"], r["cpu_parallel_gbs"] = par, in_bytes / 1e9 / par

            # ---- in-place tree API on a fresh copy, checked against the reference-stripped tree
            def tree():
                run = os.path.join(base, "gpu")
                shutil.rmtree(run, ignore_errors=True)
                shutil.copytree(master, run, symlinks=True)
                t0 = time.perf_counter()
                st = S.strip_tree(run, ctx=ctx)
                dt = time.perf_counter() - t0
                tree.st = st
                return dt

            cold = N.Context(0)           # a fresh context: first call pays the pinned-arena allocation, like a one-shot CLI run
            try:
                def tree_cold():
                    run = os.path.join(base, "gpu")
                    shutil.rmtree(run, ignore_errors=True)
                    shutil.copytree(master, run, symlinks=True)
                    t0 = time.perf_counter()
                    S.strip_tree(run, ctx=cold)
                    return time.perf_counter() - t0
                r["tree_cold_first_call_s"] = tree_cold()
            finally:
                cold.close()
            tt, tts = best(tree, 3)
            gpu_snap = snapshot(os.path.join(base, "gpu"))
            r["tree_identical_to_reference"] = (gpu_snap == ref_snap)
            r["tree_s"], r["tree_gbs"] = tt, in_bytes / 1e9 / tt
            r["tree_stats"] = {k: tree.st[k] for k in ("n_gpu", "n_fallback", "n_failed", "walk_read_s", "gpu_s", "write_s")}

            # ---- device resident
            blobs = [open(p, "rb").read() for p in files]
            b = DeviceBatch.from_blobs(ctx, blobs)
            for _ in range(5):
                b.strip_async(); st = b.results()
            plan, comp, wall = [], [], []
            for _ in range(20):
                t0 = time.perf_counter()
                b.strip_async(); st = b.results()
                wall.append(time.perf_counter() - t0)
                plan.append(st["plan_ms"]); comp.append(st["compact_ms"])
            alg = st["copy_bytes"] + st["out_bytes"]
            r["device"] = {"n_ok": st["n_ok"], "n_unsupported": st["n_unsupported"], "plan_ms": float(np.median(plan)), "compact_ms": float(np.median(comp)),
                           "step_ms_wall": float(np.median(wall)) * 1e3, "gbs_input": in_bytes / 1e9 / (float(np.median(wall))),
                           "kernels_gbs_input": in_bytes / 1e9 / ((float(np.median(plan)) + float(np.median(comp))) / 1e3),
                           "compact_rw_gbs": alg / 1e9 / (float(np.median(comp)) / 1e3), "compact_frac": alg / 1e9 / (float(np.median(comp)) / 1e3) / peak,
                           "copy_bytes": st["copy_bytes"], "out_bytes": st["out_bytes"], "header_bytes": st["header_bytes"]}
            b.close()
            # ---- host buffers
            ts = []
            for i in range(6):
                t0 = time.perf_counter()
                outs, status, hst = S.strip_buffers(ctx, blobs)
                ts.append(time.perf_counter() - t0)
            r["host_api_note"] = "strip_buffers incl. pinned allocation and Python packing; see bench.py e2e for the steady-state figure"
            r["host_api_s"] = min(ts)
            res["trees"][name] = r
            sys.stderr.write("%s: %s\n" % (name, json.dumps({k: v for k, v in r.items() if k not in ("tree_stats",)})[:400]))
    finally:
        shutil.rmtree(base, ignore_errors=True)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
