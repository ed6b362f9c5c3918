"""zip_build(check=...) against zip_build followed by check_zip on the zip it wrote.

Workloads: the installed numpy and scipy as two wheels ("numpy_scipy_wheels") and as two tarballs written by tarfile
"w:gz" ("numpy_scipy_tarballs"), each written with and without seek tables in the zip ("_zst"), and each checked
without and with symbols=True (mount /opt, prefix "python/").  The CUDA context is created and every engine warmed up
before any clock starts; then, per configuration, one warm-up pair and three alternating runs of the two routes.  The
reports of the two routes are compared (everything but the timings and bus bytes).  Recorded: the card's name, power
limit and clock, the end-to-end times (median of three), the check's kernel time (parse and symbol kernels, CUDA
events), the inflate kernel time the check spent (the writer's: only round-two wheel members; check_zip's: every
object), and the bytes each check moved over the bus.  One JSON line per configuration is printed and appended to
--out.

    python tools/measure_layer_check.py [--out results/h100_layer_check.jsonl]
"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tarfile
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from lambdipy_b200 import _native as N  # noqa: E402
from lambdipy_b200 import deps, layer  # noqa: E402
from measure_gzip import gpu_info  # noqa: E402
from measure_zip_tarballs import sm_clock  # noqa: E402
from test_gpu_layer_build import SITE, installed_wheel  # noqa: E402

STAT_KEYS = ("members", "roots", "objects", "rounds", "references", "lookups", "symbols_skipped")


def tarballs(tmp):
    out = []
    for name in ("numpy", "scipy"):
        p = os.path.join(tmp, name + ".tar.gz")
        with tarfile.open(p, "w:gz") as tar:
            for d in (name, name + ".libs"):
                if os.path.exists(os.path.join(SITE, d)):
                    tar.add(os.path.join(SITE, d), arcname=d)
        out.append(p)
    return out


def comparable(rep):
    return ({k: v for k, v in rep.items() if k != "stats"}, {k: rep["stats"].get(k) for k in STAT_KEYS})


def measure(ctx, case, srcs, tmp, seek, symbols):
    tars, wheels = (srcs, ()) if case.endswith("tarballs") else ((), srcs)
    check = {"mount": "/opt", "symbols": symbols}
    dst = os.path.join(tmp, "layer.zip")
    kw = {"prefix": "python/", "ctx": ctx, "seek_table": seek}

    def inline():
        t0 = time.perf_counter()
        st = layer.zip_build(dst, tars, wheels, check=check, **kw)
        return time.perf_counter() - t0, st["check"]

    def after():
        t0 = time.perf_counter()
        layer.zip_build(dst, tars, wheels, **kw)
        rep = deps.check_zip(dst, ctx=ctx, **check)
        return time.perf_counter() - t0, rep

    inline()
    after()
    a, b = [], []
    for _ in range(3):
        a.append(inline())
        b.append(after())
    ra, rb = a[-1][1], b[-1][1]
    sa, sb = ra["stats"], rb["stats"]
    kernel = lambda s: s["parse_ms"] + s.get("symbols_ms", 0.0)  # noqa: E731
    out = {"case": case + ("_zst" if seek else ""), "symbols": symbols, "gpu": gpu_info(), "sm_clock": sm_clock(),
           "reports_equal": comparable(ra) == comparable(rb), "problems": len(ra["problems"]),
           "roots": sa["roots"], "roots_reused": sa["roots_reused"], "objects": sa["objects"], "rounds": sa["rounds"],
           "e2e_zip_build_check_s": round(statistics.median(t for t, _ in a), 3),
           "e2e_zip_build_then_check_zip_s": round(statistics.median(t for t, _ in b), 3),
           "runs_zip_build_check_s": [round(t, 3) for t, _ in a],
           "runs_zip_build_then_check_zip_s": [round(t, 3) for t, _ in b],
           "check_kernel_ms": round(kernel(sa), 3), "check_zip_kernel_ms": round(kernel(sb), 3),
           "check_inflate_ms": round(sa["inflate_ms"], 3), "check_zip_inflate_ms": round(sb["inflate_ms"], 3),
           "check_bytes_up": sa["bytes_up"], "check_bytes_down": sa["bytes_down"],
           "check_zip_bytes_up": sb["bytes_up"], "check_zip_bytes_down": sb["bytes_down"]}
    out["saved_s"] = round(out["e2e_zip_build_then_check_zip_s"] - out["e2e_zip_build_check_s"], 3)
    if symbols:
        out.update({"references": sa["references"], "lookups": sa["lookups"]})
    os.remove(dst)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_layer_check.jsonl"))
    args = ap.parse_args()
    with N.Context(0) as ctx:   # no device: this raises, nothing is timed
        tmp = tempfile.mkdtemp(prefix="lb2_layer_check_")
        try:
            wdir = os.path.join(tmp, "wheels")
            os.makedirs(wdir)
            cases = {"numpy_scipy_wheels": [installed_wheel(d, wdir) for d in ("numpy", "scipy")],
                     "numpy_scipy_tarballs": tarballs(tmp)}
            warm = os.path.join(tmp, "warm.zip")
            for case, srcs in cases.items():     # module load and first allocations of every engine
                tars, wheels = (srcs[:1], ()) if case.endswith("tarballs") else ((), srcs[:1])
                layer.zip_build(warm, tars, wheels, ctx=ctx)
                deps.check_zip(warm, ctx=ctx, symbols=True)
                try:
                    layer.zip_build(warm, tars, wheels, ctx=ctx, check={"symbols": True})
                except deps.CheckFailed:
                    pass
            for case, srcs in cases.items():
                for seek in (False, True):
                    for symbols in (False, True):
                        line = json.dumps(measure(ctx, case, srcs, tmp, seek, symbols))
                        print(line, flush=True)
                        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                        with open(args.out, "a") as f:
                            f.write(line + "\n")
        finally:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
