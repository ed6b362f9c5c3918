"""lb2_syms_find and check_zip(python=...) on the H100, against the emulator of the same logic
(tests/emu/syms_find_emu.cpp) and check_with behind zlib and the emulators:

* find's records equal the emulator's on the CPU corpus and the PyInit fixtures, each object at an odd device
  address and freed before the lookups, with queries over single objects and over whole closures;
* check_zip(python="3.12") equals check_with on numpy + scipy zipped by make_archive and by zip_tree(seek_table=True);
* zip_build(check={"python": "3.12"}) gives check_zip's report of the zip written, and a renamed module raises
  CheckFailed with no dst;
* python=None gives the same stats and bus bytes as before; a second run gives the same report; only the names go up
  beyond the arrays, and only the found records come down;
* LB2_E_CAPACITY in the index still halves its batches."""
import ctypes
import os

import pytest

import deps_lib as D
import find_lib as FL
from lambdipy_b200 import _native as N
from lambdipy_b200 import deps
from lambdipy_b200 import layer as L
from lambdipy_b200 import zipfile_gpu as Z
from test_gpu_elf_syms import _without_stats, layer_zips  # noqa: F401  (fixture)
from test_gpu_layer_check import _CapacityCtx
from test_layer_build_host import whl
from test_python_imports_emulated import fx  # noqa: F401  (fixture)
from test_python_imports_host import MOD, T312, _cc
from test_python_imports_host import check as host_check

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    with N.Context(0) as c:
        yield c


@pytest.fixture(scope="module")
def emu():
    return D.Emu()


def _queries(idx, names):
    """each name in each object alone, then in the scope of all objects"""
    ids = [i for i, _, _ in idx]
    queries = [(k, 1, n) for k in range(len(ids)) for n in names] + [(0, len(ids), n) for n in names]
    return queries, ids


def test_find_equals_emulator(ctx, fx, tmp_path):  # noqa: F811
    corpus = D.corpus(str(tmp_path))
    files = sorted(corpus.values()) + sorted({p for m, more, _ in fx.values() for p in [m] + more})
    blobs = []
    for p in files:
        with open(p, "rb") as f:
            blobs.append(f.read())
    names = sorted({n.encode() for _, _, n in fx.values()} | {b"PyInit__multiarray_umath", b"malloc", b"a_val", b"v1",
                                                               b"", b"x" * 300})
    emu = FL.EmuResolver()
    idx = emu.index_blobs(blobs)
    queries, ids = _queries(idx, names)
    want = emu.find(queries, ids)
    bufs, refs = [], []
    for b in blobs:
        p = ctx.dev_alloc(len(b) + 32)
        bufs.append(p)
        if b:
            ctx.h2d(p + 3, b, len(b))
        refs.append((p + 3, len(b)))
    with deps.GpuSymbolResolver(ctx) as r:
        gidx = r.index(refs)
        for p in bufs:  # the arena must not need the objects any more
            ctx.dev_free(p)
        assert [g[1:] for g in gidx] == [e[1:] for e in idx]
        got = r.find(queries, [i for i, _, _ in gidx])
        assert got == want
        assert sum(1 for g in got if g[0] is not None) > len(fx)
        # bus bytes: the objects' records, the queries, the scope and the names up; the found records down
        up0, down0 = r.uploaded, r.downloaded
        r.find(queries, ids)
        pool = sum(len(q[2]) for q in queries)
        assert r.uploaded - up0 == ctypes.sizeof(N.SymObject) * len(gidx) + 16 * len(queries) + 4 * len(ids) + pool
        assert r.downloaded - down0 == 12 * len(queries)
        assert r.stats()["find_queries"] == 2 * len(queries) and r.stats()["find_ms"] > 0
        assert r.find([], ids) == []
        with pytest.raises(N.NativeError):
            r.find([(0, len(ids) + 1, b"x")], ids)


def test_check_zip_python_numpy_scipy(ctx, emu, layer_zips):  # noqa: F811
    for label, z in layer_zips.items():
        plain = deps.check_zip(z, mount="/opt", ctx=ctx)
        rep = deps.check_zip(z, mount="/opt", ctx=ctx, python="3.12")
        want = host_check(z, emu, mount="/opt", python="3.12")
        assert _without_stats(rep) == _without_stats(want), label
        assert [p for p in rep["problems"] if p["kind"] == "python"] == []
        st = rep["stats"]
        for k in ("modules", "python_skipped", "find_queries", "objects", "rounds"):
            assert st[k] == want["stats"][k], (label, k)
        assert st["modules"] > 50 and st["find_ms"] > 0
        assert _without_stats(deps.check_zip(z, mount="/opt", ctx=ctx, python="3.12")) == _without_stats(rep)
        old = deps.check_zip(z, mount="/opt", ctx=ctx, python="3.11")
        assert _without_stats(old) == _without_stats(host_check(z, emu, mount="/opt", python="3.11"))
        tagged = {p for p in rep["python"]["modules"] if ".cpython-" in p.rsplit("/", 1)[1]}
        old_problems = {p["object"] for p in old["problems"] if p["kind"] == "python"}
        assert old_problems <= tagged and len(old_problems) > 50
        # python=None: the stats and bus bytes of the check without the option, timings aside
        again = deps.check_zip(z, mount="/opt", ctx=ctx)
        assert _without_stats(again) == _without_stats(plain)
        for k in ("members", "roots", "objects", "rounds", "bytes_up", "bytes_down"):
            assert again["stats"][k] == plain["stats"][k], (label, k)
        assert "python" not in plain and "modules" not in plain["stats"]
        both = deps.check_zip(z, mount="/opt", ctx=ctx, python="3.12", symbols=True)
        assert both["python"] == rep["python"] and "symbols" in both


def _wheel(d, name, files):
    out = []
    for member, src in files.items():
        with open(src, "rb") as f:
            out.append((member, f.read(), 0o755))
    return whl(os.path.join(d, "%s-1.0-py3-none-any.whl" % name), name, "1.0", out, (2024, 1, 1, 0, 0, 0))


def test_zip_build_check_python(ctx, tmp_path):
    d = str(tmp_path)
    good, renamed = _cc(d, "good.so", MOD % "good"), _cc(d, "renamed.so", MOD % "original")
    w_good = _wheel(d, "good", {"good" + T312: good})
    dst = os.path.join(d, "layer.zip")
    check = {"mount": "/opt", "python": "3.12"}
    st = L.zip_build(dst, (), [w_good], prefix="python/", ctx=ctx, check=check)
    want = deps.check_zip(dst, ctx=ctx, **check)
    assert _without_stats(st["check"]) == _without_stats(want)
    assert st["check"]["python"]["modules"]["/opt/python/good" + T312]["status"] == "ok" and want["problems"] == []
    w_bad = _wheel(d, "bad", {"renamed" + T312: renamed})
    bad = os.path.join(d, "bad.zip")
    with pytest.raises(deps.CheckFailed) as e:
        L.zip_build(bad, (), [w_bad], prefix="python/", ctx=ctx, check=check)
    assert not os.path.exists(bad) and "PyInit_renamed not exported" in str(e.value)


def test_capacity_halves_the_index(ctx, layer_zips):  # noqa: F811
    z = layer_zips["make_archive"]
    want = deps.check_zip(z, mount="/opt", ctx=ctx, python="3.12")
    cap = _CapacityCtx(ctx)
    with deps.GpuSymbolResolver(cap) as r, Z.GpuUnzipDecoder(ctx) as dec, deps.GpuElfParser(ctx) as parser:
        got = deps.check_with(z, dec, parser, mount="/opt", python="3.12", resolver=r)
    assert cap.lib.refused > 0 and _without_stats(got) == _without_stats(want)
