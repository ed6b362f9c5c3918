"""lb2_elf_deps and check_zip on the H100, against the emulator of the same parse (tests/emu/deps_emu.cpp) and
check_with behind zlib and that emulator:

* the kernel's records equal the emulator's on the whole CPU corpus and on the mutants;
* check_zip on numpy + scipy zipped by make_archive and by zip_tree (with and without seek tables) equals check_with,
  reaches the .libs targets in 3 rounds and reports GLIBC_2.27 as the highest glibc need;
* a torch/lib zip reports the CUDA libraries as missing;
* bytes up are the parsed members' bodies, bytes down only objects, records and pool;
* halving on LB2_E_CAPACITY gives the same report, and so does a second run."""
import os
import shutil
import zipfile

import pytest

import deps_lib as D
import elf_fixtures as F
import elf_mutants as M
from lambdipy_b200 import _native as N
from lambdipy_b200 import deps
from lambdipy_b200 import zipfile_gpu as Z
from test_deps_host import check as host_check

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    with N.Context(0) as c:
        yield c


@pytest.fixture(scope="module")
def emu():
    return D.Emu()


def gpu_parse(ctx, blobs):
    """each blob uploaded to its own device buffer at an odd address (byte alignment only), parsed in one batch"""
    bufs, refs = [], []
    for b in blobs:
        p = ctx.dev_alloc(len(b) + 32)
        bufs.append(p)
        if b:
            ctx.h2d(p + 3, b, len(b))
        refs.append((p + 3, len(b)))
    try:
        with deps.GpuElfParser(ctx) as parser:
            return parser.parse(refs)
    finally:
        for p in bufs:
            ctx.dev_free(p)


def test_kernel_equals_emulator_on_corpus_and_mutants(ctx, emu, tmp_path):
    corpus = D.corpus(str(tmp_path))
    blobs = []
    for k in sorted(corpus):
        with open(corpus[k], "rb") as f:
            blobs.append(f.read())
    assert gpu_parse(ctx, blobs) == emu.parse(blobs)
    for bi, k in enumerate(("variant/c_rpath_soname", "linked/libuser_rpath.so", "linked/libv.so",
                            "golden/real_libXau.in.bin")):
        with open(corpus[k], "rb") as f:
            data = f.read()
        ms = [m for _, m in M.mutants(data, bi)] + [data[:n] for n in range(0, len(data), 97)]
        assert gpu_parse(ctx, ms) == emu.parse(ms), k


def _layer_tree(root):
    sp = F.site_packages()
    for r in ("numpy", "scipy", "numpy.libs", "scipy.libs"):
        shutil.copytree(os.path.join(sp, r), os.path.join(root, "python", r), symlinks=True,
                        ignore=shutil.ignore_patterns("__pycache__", "tests"))
    return root


@pytest.fixture(scope="module")
def layer_zips(tmp_path_factory, ctx):
    d = tmp_path_factory.mktemp("np_layer")
    tree = _layer_tree(str(d / "tree"))
    out = {"make_archive": shutil.make_archive(str(d / "ma"), "zip", tree)}
    for seek in (False, True):
        p = str(d / ("zt%d.zip" % seek))
        Z.zip_tree(tree, p, ctx=ctx, **({"seek_table": True} if seek else {}))
        out["zip_tree%s" % ("_seek" if seek else "")] = p
    return out


def _without_stats(rep):
    return {k: v for k, v in rep.items() if k != "stats"}


def test_check_zip_numpy_scipy_layer(ctx, emu, layer_zips):
    for label, z in layer_zips.items():
        rep = deps.check_zip(z, mount="/opt", ctx=ctx)
        want = host_check(z, emu, mount="/opt")
        assert _without_stats(rep) == _without_stats(want), label
        st = rep["stats"]
        assert st["rounds"] == 3 and rep["max_versions"]["GLIBC"] == "2.27" and rep["problems"] == [], label
        assert any("numpy.libs/libgfortran" in p for p in rep["objects"]) and \
            any("numpy.libs/libquadmath" in p for p in rep["objects"])
        # up: the parsed members' bodies; down: objects, records and pool
        with zipfile.ZipFile(z) as zf:
            parsed = {rep["objects"][p]["member"] for p in rep["objects"]}
            assert st["bytes_up"] == sum(zf.getinfo(m).compress_size for m in parsed), label
        n_rec = sum(len(o["needed"] or []) for o in rep["objects"].values())
        assert st["bytes_down"] < 64 * st["objects"] + 64 * 1024 + 200 * n_rec, label
        assert st["parse_ms"] > 0 and st["inflate_ms"] > 0
        assert _without_stats(deps.check_zip(z, mount="/opt", ctx=ctx)) == _without_stats(rep)  # deterministic


def test_check_zip_halving_gives_the_same_report(ctx, layer_zips):
    z = layer_zips["make_archive"]
    want = deps.check_zip(z, mount="/opt", ctx=ctx)

    class Halving(Z.GpuUnzipDecoder):
        """refuses any run of more than 8 members, as a device too small for them would"""
        refused = 0

        def run(self, n, members, device=False, tables=None):
            if len(members) > 8:
                Halving.refused += 1
                raise Z.DeviceTooSmall("LB2_E_CAPACITY")
            return super().run(n, members, device=device, tables=tables)

    with Halving(ctx) as dec, deps.GpuElfParser(ctx) as parser:
        got = deps.check_with(z, dec, parser, mount="/opt")
    assert Halving.refused > 0
    assert _without_stats(got) == _without_stats(want)


def test_torch_lib_reports_cuda_libraries_missing(ctx, tmp_path):
    sp = F.site_packages()
    lib = os.path.join(sp, "torch", "lib")
    if not os.path.isdir(lib):
        pytest.skip("torch/lib is not installed here")
    z = str(tmp_path / "torchlib.zip")
    with zipfile.ZipFile(z, "w", zipfile.ZIP_STORED) as zf:  # stored: the test is about the closure, not the inflate
        for name in sorted(os.listdir(lib)):
            if not os.path.islink(os.path.join(lib, name)) and os.path.isfile(os.path.join(lib, name)):
                zf.write(os.path.join(lib, name), "lib/" + name)
    rep = deps.check_zip(z, mount="/opt/python/torch", ctx=ctx)
    missing = {p["detail"].split(":")[0] for p in rep["problems"] if p["kind"] == "missing"}
    assert {"libcudart.so.12", "libcublas.so.12"} <= missing, sorted(missing)
    assert any(m.startswith("libcudnn.so") for m in missing)
