"""lb2_syms_* and check_zip(symbols=True) on the H100, against the emulator of the same logic (tests/emu/syms_emu.cpp)
and check_with behind zlib and the emulators:

* the kernels' index, lookups and miss names equal the emulator's on the CPU corpus and on mutants, each object at an
  odd device address;
* check_zip(symbols=True) equals check_with with the emulators on numpy + scipy zipped by make_archive and by
  zip_tree(seek_table=True), and on torch/lib;
* a library rebuilt without one symbol, zipped with its user, is reported;
* a second run gives the same report; bytes down grow only by counts, misses and their names;
* halving the decoder's batches and growing the miss buffer give the same report;
* symbols=False gives the report check_zip gave before the option existed."""
import os
import shutil
import subprocess
import sys
import zipfile

import pytest

import deps_lib as D
import elf_fixtures as F
import syms_lib as S
from lambdipy_b200 import _native as N
from lambdipy_b200 import deps
from lambdipy_b200 import zipfile_gpu as Z
from test_deps_host import make_zip
from test_elf_syms_emulated import symbol_mutants
from test_symbols_host import check as host_check

pytestmark = pytest.mark.gpu
HOST_LIBS = "/lib/x86_64-linux-gnu"


@pytest.fixture(scope="module")
def ctx():
    with N.Context(0) as c:
        yield c


@pytest.fixture(scope="module")
def emu():
    return D.Emu()


def _all_in_all(r, n_ids, ids):
    """index, then every object's references resolved in the scope of all of them: (index, counts, misses, names)"""
    jobs = [(i, 0, len(ids)) for i in ids]
    classes = [k % 3 for k in range(n_ids)]
    counts, misses = r.resolve(jobs, ids, classes)
    return counts, misses, r.names(jobs, misses)


def gpu_run(ctx, blobs):
    bufs, refs = [], []
    for b in blobs:
        p = ctx.dev_alloc(len(b) + 32)
        bufs.append(p)
        if b:
            ctx.h2d(p + 3, b, len(b))
        refs.append((p + 3, len(b)))
    try:
        with deps.GpuSymbolResolver(ctx) as r:
            idx = r.index(refs)
            for p in bufs:  # the arena must not need the objects any more
                ctx.dev_free(p)
            bufs = []
            return idx, _all_in_all(r, len(idx), [i for i, _, _ in idx])
    finally:
        for p in bufs:
            ctx.dev_free(p)


def emu_run(blobs):
    r = S.EmuResolver()
    idx = r.index_blobs(blobs)
    return idx, _all_in_all(r, len(idx), [i for i, _, _ in idx])


def test_kernels_equal_emulator_on_corpus_and_mutants(ctx, tmp_path):
    corpus = D.corpus(str(tmp_path))
    blobs = []
    for k in sorted(corpus):
        with open(corpus[k], "rb") as f:
            blobs.append(f.read())
    got = gpu_run(ctx, blobs)
    assert got == emu_run(blobs)
    assert sum(n for _, _, n in got[0]) > 10000 and got[1][1]
    for bi, k in enumerate(("golden/c_plain.in.bin", "linked/libv.so", "linked/libuser_rpath.so")):
        with open(corpus[k], "rb") as f:
            data = f.read()
        ms = [m for _, m in symbol_mutants(data, bi)] + [data[:n] for n in range(0, len(data), 211)]
        assert gpu_run(ctx, ms) == emu_run(ms), k


def _layer_tree(root):
    sp = F.site_packages()
    for r in ("numpy", "scipy", "numpy.libs", "scipy.libs"):
        shutil.copytree(os.path.join(sp, r), os.path.join(root, "python", r), symlinks=True,
                        ignore=shutil.ignore_patterns("__pycache__", "tests"))
    return root


@pytest.fixture(scope="module")
def layer_zips(tmp_path_factory, ctx):
    d = tmp_path_factory.mktemp("np_syms")
    tree = _layer_tree(str(d / "tree"))
    out = {"make_archive": shutil.make_archive(str(d / "ma"), "zip", tree)}
    p = str(d / "zt_seek.zip")
    Z.zip_tree(tree, p, ctx=ctx, seek_table=True)
    out["zip_tree_seek"] = p
    return out


def _without_stats(rep):
    return {k: v for k, v in rep.items() if k != "stats"}


KW = {"interpreter": [sys.executable], "runtime_libs": [HOST_LIBS]}


def test_check_zip_symbols_numpy_scipy(ctx, emu, layer_zips):
    for label, z in layer_zips.items():
        plain = deps.check_zip(z, mount="/opt", ctx=ctx)
        for kw in ({}, KW):
            rep = deps.check_zip(z, mount="/opt", ctx=ctx, symbols=True, **kw)
            want = host_check(z, emu, mount="/opt", **kw)
            assert _without_stats(rep) == _without_stats(want), (label, kw)
            assert rep["problems"] == [], rep["problems"][:3]
            st = rep["stats"]
            assert st["references"] == want["stats"]["references"] and st["lookups"] == want["stats"]["lookups"]
            assert st["symbols_ms"] > 0 and st["symbols_resolve_ms"] > 0
            assert _without_stats(deps.check_zip(z, mount="/opt", ctx=ctx, symbols=True, **kw)) == _without_stats(rep)
            # down: the deps records as before, plus per-object index records, counts, misses and their names
            assert st["bytes_down"] - plain["stats"]["bytes_down"] < 1024 * (st["objects"] + 64) + 64 * st["references"]
            assert st["bytes_up"] >= plain["stats"]["bytes_up"]
        # symbols=False: the report of check_zip without the option
        assert set(plain) == {"arch", "mount", "objects", "closures", "resolved", "problems", "notes", "max_versions",
                              "provided_used", "stats"}
        assert set(plain["stats"]) == {"members", "roots", "objects", "rounds", "bytes_up", "bytes_down", "inflate_ms",
                                       "parse_ms"}


def test_halving_and_miss_buffer_growth(ctx, layer_zips):
    z = layer_zips["make_archive"]
    want = deps.check_zip(z, mount="/opt", ctx=ctx, symbols=True)

    class Halving(Z.GpuUnzipDecoder):
        refused = 0

        def run(self, n, members, device=False, tables=None):
            if len(members) > 8:
                Halving.refused += 1
                raise Z.DeviceTooSmall("LB2_E_CAPACITY")
            return super().run(n, members, device=device, tables=tables)

    with Halving(ctx) as dec, deps.GpuElfParser(ctx) as parser, deps.GpuSymbolResolver(ctx) as r:
        r._miss_cap = 1
        got = deps.check_with(z, dec, parser, mount="/opt", symbols=True, resolver=r)
        assert r._miss_cap > 1
    assert Halving.refused > 0 and _without_stats(got) == _without_stats(want)


def test_torch_lib(ctx, emu, tmp_path):
    lib = os.path.join(F.site_packages(), "torch", "lib")
    if not os.path.isdir(lib):
        pytest.skip("torch/lib is not installed here")
    z = str(tmp_path / "torchlib.zip")
    with zipfile.ZipFile(z, "w", zipfile.ZIP_STORED) as zf:
        for name in sorted(os.listdir(lib)):
            if not os.path.islink(os.path.join(lib, name)) and os.path.isfile(os.path.join(lib, name)):
                zf.write(os.path.join(lib, name), "lib/" + name)
    rep = deps.check_zip(z, mount="/opt/python/torch", ctx=ctx, symbols=True, **KW)
    want = host_check(z, emu, mount="/opt/python/torch", **KW)
    assert _without_stats(rep) == _without_stats(want)
    assert rep["stats"]["references"] > 0 or rep["stats"]["symbols_skipped"] == rep["stats"]["roots"]


def test_rebuilt_library_without_a_symbol_is_reported(ctx, tmp_path):
    d = str(tmp_path)

    def cc(out, code, *args):
        src = os.path.join(d, out + ".cc")
        with open(src, "w") as f:
            f.write(code)
        subprocess.run(["g++", "-shared", "-fPIC", "-O1", "-o", os.path.join(d, out), src] + list(args), check=True)
        return os.path.join(d, out)
    core = "namespace c10 { struct RegisterOperators { RegisterOperators(); int op(int); };\n" \
           "RegisterOperators::RegisterOperators() {}\n%s }\n"
    new = cc("libcore.so", core % "int RegisterOperators::op(int x) { return x; }", "-Wl,-soname,libcore.so")
    old = cc("libcore_old.so", core % "", "-Wl,-soname,libcore.so")
    user = cc("_C.so", "namespace c10 { struct RegisterOperators { RegisterOperators(); int op(int); }; }\n"
                       "int reg(void) { c10::RegisterOperators r; return r.op(1); }\n", "-L" + d, "-lcore",
              "-Wl,-rpath,$ORIGIN/lib")
    ok = make_zip(str(tmp_path / "ok.zip"), {"pkg/_C.so": user, "pkg/lib/libcore.so": new})
    bad = make_zip(str(tmp_path / "bad.zip"), {"pkg/_C.so": user, "pkg/lib/libcore.so": old})
    assert deps.check_zip(ok, ctx=ctx, symbols=True, **KW)["problems"] == []
    rep = deps.check_zip(bad, ctx=ctx, symbols=True, **KW)
    assert [(p["object"], p["kind"], p["detail"]) for p in rep["problems"]] == [
        ("/var/task/pkg/_C.so", "symbol",
         "_ZN3c1017RegisterOperators2opEi: no definition in the load scope of /var/task/pkg/_C.so")]
    assert deps.check_zip(bad, ctx=ctx)["problems"] == []  # the check without symbols passes it
