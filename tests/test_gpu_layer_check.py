"""GPU checks of zip_build(check=...) and zip_tarballs(check=...): the check run on the H100 over the objects the
writer holds in device memory, before the zip is written.

The oracle is check_zip on the zip that was written: the report must be the same, apart from the engine timings and
bus bytes in stats.  Cases: numpy + scipy as two wheels (prefix "python/", mount /opt, symbols with the interpreter
and the host's libraries), numpy as a tarball with scipy as a wheel, and zip_tarballs of the gcc variants with links
and the golden files.  Also: the zip is byte for byte the zip written without the check; a C++ library rebuilt
without a member function, inside a wheel, raises CheckFailed naming it and writes nothing; every root is checked
where the build left it and only round-two wheel bodies, the interpreter and the runtime files go up; LB2_E_CAPACITY
forced in the decoder and in the symbol resolver gives the same report; a second run gives the same report."""
import gzip
import io
import os
import shutil
import subprocess
import sys
import tarfile
import zipfile

import numpy as np
import pytest

from test_gpu_layer_build import D1, installed_wheel, whl
from test_gpu_strip_tarball import GOLDEN, variant_tree, write_tgz

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))
HOST_LIBS = "/lib/x86_64-linux-gnu"
FULL = {"mount": "/opt", "symbols": True, "interpreter": [sys.executable], "runtime_libs": [HOST_LIBS]}
STAT_KEYS = ("members", "roots", "objects", "rounds", "references", "lookups", "symbols_skipped")


def same(got, want):
    assert {k: v for k, v in got.items() if k != "stats"} == {k: v for k, v in want.items() if k != "stats"}
    assert {k: got["stats"].get(k) for k in STAT_KEYS} == {k: want["stats"].get(k) for k in STAT_KEYS}


@pytest.fixture(scope="module")
def wheels(tmp_path_factory):
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    d = str(tmp_path_factory.mktemp("check_wheels"))
    return installed_wheel("numpy", d), installed_wheel("scipy", d)


class _CapacityLib:
    """the native library with lb2_syms_index refusing batches of more than 4 objects (LB2_E_CAPACITY)"""

    def __init__(self, lib):
        self._lib, self.refused = lib, 0

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def lb2_syms_index(self, h, ptrs, sizes, n, *rest):
        from lambdipy_b200 import _native as N
        if n > 4:
            self.refused += 1
            return N.LB2_E_CAPACITY
        return self._lib.lb2_syms_index(h, ptrs, sizes, n, *rest)


class _CapacityCtx:
    def __init__(self, ctx):
        self._ctx, self.lib = ctx, _CapacityLib(ctx.lib)

    def __getattr__(self, name):
        return getattr(self._ctx, name)


def build(ctx, dst, tarballs, wheels, check, prefix="python/", decoder=None, resolver_ctx=None, seek_table=False):
    """zip_build's engines by hand, so that the parser's and the resolver's uploads can be read: (stats, bytes the
    parser uploaded, bytes the resolver uploaded)"""
    from lambdipy_b200 import deps as D
    from lambdipy_b200 import layer as L
    from lambdipy_b200 import tarball as T
    from lambdipy_b200 import zipfile_gpu as Z
    with T.GpuTarReader(ctx) as reader, (decoder or Z.GpuUnzipDecoder)(ctx) as dec, Z.GpuStripper(ctx) as stripper, \
            Z.GpuZipEncoder(ctx, L.PIECE_BYTES, host_buffers=False, seek_table=seek_table) as enc, D.GpuElfParser(ctx) as parser, \
            D.GpuSymbolResolver(resolver_ctx or ctx) as resolver:
        st = L.build_with(dst, tarballs, wheels, reader, T.GpuTarIndex(ctx), dec, stripper, enc, prefix, check=check,
                          parser=parser, resolver=resolver if check.get("symbols") else None)
        return st, parser.uploaded, resolver.uploaded


def later_wheel_bodies(report, dst, wheels, prefix):
    """the compressed bodies of the objects a closure reached that are not roots and come from a wheel"""
    names = set()
    for w in wheels:
        names |= {prefix + n for n in zipfile.ZipFile(w).namelist()}
    with zipfile.ZipFile(dst) as zf:
        return sum(zf.getinfo(o["member"]).compress_size for o in report["objects"].values()
                   if not o["member"].rsplit("/", 1)[-1].endswith(".so") and o["member"] in names)


def test_numpy_scipy_wheels(gpu_ctx, tmp_path, wheels):
    from lambdipy_b200 import deps as D
    from lambdipy_b200 import layer as L
    plain = str(tmp_path / "plain.zip")
    L.zip_build(plain, (), wheels, prefix="python/", ctx=gpu_ctx)
    dst = str(tmp_path / "layer.zip")
    st, parser_up, resolver_up = build(gpu_ctx, dst, (), wheels, FULL)
    assert open(dst, "rb").read() == open(plain, "rb").read()
    rep = st["check"]
    want = D.check_zip(dst, ctx=gpu_ctx, **FULL)
    same(rep, want)
    assert rep["problems"] == [] and rep["stats"]["rounds"] >= 2 and rep["stats"]["objects"] > rep["stats"]["roots"]
    s = rep["stats"]
    later = later_wheel_bodies(rep, dst, wheels, "python/")
    assert s["roots_reused"] == s["roots"] > 100 and later > 0
    # up: the round-two wheel bodies, the interpreter's and the runtime's files (the parser's uploads), and the
    # resolver's job arrays; no root
    assert s["bytes_up"] == later + parser_up + resolver_up and parser_up >= os.path.getsize(os.path.realpath(sys.executable))
    assert s["symbols_ms"] > 0 and s["parse_ms"] > 0 and s["inflate_ms"] > 0
    # without symbols, only the round-two bodies go up
    plain_check = dict(FULL, symbols=False)
    st2 = L.zip_build(str(tmp_path / "l2.zip"), (), wheels, prefix="python/", ctx=gpu_ctx, check=plain_check)
    assert st2["check"]["stats"]["bytes_up"] == later
    same(st2["check"], D.check_zip(dst, ctx=gpu_ctx, **plain_check))
    # a second run, and LB2_E_CAPACITY forced in the decoder and in the resolver
    from lambdipy_b200 import zipfile_gpu as Z

    class Halving(Z.GpuUnzipDecoder):
        refused = 0

        def run(self, n, members, device=False, tables=None):
            if len(members) > 2:
                Halving.refused += 1
                raise Z.DeviceTooSmall("LB2_E_CAPACITY")
            return super().run(n, members, device=device, tables=tables)
    cap = _CapacityCtx(gpu_ctx)
    st3, _, _ = build(gpu_ctx, str(tmp_path / "l3.zip"), (), wheels, FULL, decoder=Halving, resolver_ctx=cap)
    assert Halving.refused > 0 and cap.lib.refused > 0
    assert open(str(tmp_path / "l3.zip"), "rb").read() == open(plain, "rb").read()
    same(st3["check"], rep)
    st4 = L.zip_build(str(tmp_path / "l4.zip"), (), wheels, prefix="python/", ctx=gpu_ctx, check=FULL)
    same(st4["check"], rep)


def test_numpy_tarball_scipy_wheel(gpu_ctx, tmp_path, wheels):
    from lambdipy_b200 import deps as D
    from lambdipy_b200 import layer as L
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        for d in ("numpy", "numpy.libs"):
            if os.path.exists(os.path.join(SITE, d)):
                tar.add(os.path.join(SITE, d), arcname=d)
    tgz = str(tmp_path / "numpy.tar.gz")
    with open(tgz, "wb") as f:
        f.write(gzip.compress(buf.getvalue(), compresslevel=1))
    check = {"mount": "/opt", "symbols": True}
    plain = str(tmp_path / "plain.zip")
    L.zip_build(plain, [tgz], [wheels[1]], prefix="python/", ctx=gpu_ctx, seek_table=True)
    dst = str(tmp_path / "layer.zip")
    st, parser_up, resolver_up = build(gpu_ctx, dst, [tgz], [wheels[1]], check, seek_table=True)
    assert open(dst, "rb").read() == open(plain, "rb").read()
    same(st["check"], D.check_zip(dst, ctx=gpu_ctx, **check))
    s = st["check"]["stats"]
    assert s["roots_reused"] == s["roots"] > 100 and st["check"]["problems"] == []
    # no interpreter or runtime library: the parser uploads nothing, and besides the resolver's job arrays only the
    # scipy wheel's round-two bodies go up (numpy's .libs are in the tar arena)
    assert parser_up == 0
    assert s["bytes_up"] == later_wheel_bodies(st["check"], dst, [wheels[1]], "python/") + resolver_up


def test_zip_tarballs_golden_and_variants(gpu_ctx, variants, tmp_path):
    import glob

    import tar_archives as A
    from lambdipy_b200 import deps as D
    from lambdipy_b200 import layer as L
    root = variant_tree(str(tmp_path / "pkg"), variants)
    a = write_tgz(gpu_ctx, root, str(tmp_path / "a.tar.gz"), "tarfile")
    shutil.rmtree(root)
    groot = str(tmp_path / "golden")
    A.tree(groot, {os.path.basename(p)[:-7] + ".so": open(p, "rb").read()
                   for p in sorted(glob.glob(os.path.join(GOLDEN, "*.in.bin")))})
    b = write_tgz(gpu_ctx, groot, str(tmp_path / "b.tar.gz"), "gpu")
    shutil.rmtree(groot)
    plain = str(tmp_path / "plain.zip")
    L.zip_tarballs([a, b], plain, ctx=gpu_ctx)
    for check in ({}, {"symbols": True, "runtime_libs": [HOST_LIBS]}):
        want = D.check_zip(plain, ctx=gpu_ctx, **check)
        dst = str(tmp_path / "layer.zip")
        try:
            got = L.zip_tarballs([a, b], dst, ctx=gpu_ctx, check=check)["check"]
            assert open(dst, "rb").read() == open(plain, "rb").read()
            os.remove(dst)
        except D.CheckFailed as e:                          # what check_zip says of the same zip
            got = e.report
            assert not os.path.exists(dst)
        same(got, want)
        s = got["stats"]
        assert s["roots_reused"] == s["roots"] > 10
        if not check:
            assert s["bytes_up"] == 0                        # every object was on the device already


def test_rebuilt_library_without_a_member_function(gpu_ctx, tmp_path):
    from lambdipy_b200 import deps as D
    from lambdipy_b200 import layer as L
    d = str(tmp_path)

    def cc(out, code, *args):
        src = os.path.join(d, out + ".cc")
        with open(src, "w") as f:
            f.write(code)
        subprocess.run(["g++", "-shared", "-fPIC", "-O1", "-o", os.path.join(d, out), src] + list(args), check=True)
        return open(os.path.join(d, out), "rb").read()
    core = "namespace c10 { struct RegisterOperators { RegisterOperators(); int op(int); };\n" \
           "RegisterOperators::RegisterOperators() {}\n%s }\n"
    new = cc("libcore.so", core % "int RegisterOperators::op(int x) { return x; }", "-Wl,-soname,libcore.so")
    old = cc("libcore_old.so", core % "", "-Wl,-soname,libcore.so")
    user = cc("_C.so", "namespace c10 { struct RegisterOperators { RegisterOperators(); int op(int); }; }\n"
                       "int reg(void) { c10::RegisterOperators r; return r.op(1); }\n", "-L" + d, "-lcore",
              "-Wl,-rpath,$ORIGIN/lib")
    check = {"symbols": True, "interpreter": [sys.executable], "runtime_libs": [HOST_LIBS]}
    for lib, fails in ((new, False), (old, True)):
        w = whl(os.path.join(d, "pkg-1.0-cp312-cp312-manylinux_2_17_x86_64.whl"), "pkg", "1.0",
                [("pkg/__init__.py", b"", 0o644), ("pkg/_C.so", user, 0o755), ("pkg/lib/libcore.so", lib, 0o755)], D1)
        dst = os.path.join(d, "layer.zip")
        if not fails:
            assert L.zip_build(dst, (), [w], ctx=gpu_ctx, check=check)["check"]["problems"] == []
            os.remove(dst)
            continue
        with pytest.raises(D.CheckFailed) as e:
            L.zip_build(dst, (), [w], ctx=gpu_ctx, check=check)
        assert [(p["object"], p["kind"], p["detail"]) for p in e.value.report["problems"]] == [
            ("/var/task/pkg/_C.so", "symbol",
             "_ZN3c1017RegisterOperators2opEi: no definition in the load scope of /var/task/pkg/_C.so")]
        assert "_ZN3c1017RegisterOperators2opEi" in str(e.value)
        assert not os.path.exists(dst) and not [n for n in os.listdir(d) if n.endswith(".tmp")]
