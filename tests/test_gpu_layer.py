"""GPU checks of zip_tarballs (layer.py): package tarballs to a Lambda zip, inflated, stripped and deflated on the GPU.

Parity: extract_tarball of each source into one directory (under the prefix), the real `find -name "*.so" | xargs
strip` and a walk listing every directory sorted give the entries of the zip -- names, order, types, attributes,
sizes, CRC-32 and bytes -- on gcc variants with links, the golden files, and numpy + scipy as two sources written by
tarfile "w:gz" and by gzip_tarball(seek_table=True).  The documented deviations (a stripped file keeps its mtime, a
directory without a member or added to by a later source) are applied to that tree.  Every body is zip_tree's body for
the same file of that tree, at the default level and level 9, with 64 MB and 1 MB pieces; zipfile and the GPU testzip
accept the zip; with seek_table=True extract_zip reads it from its tables; runs are deterministic; the index costs no
miss; what crosses the bus is the sources, the index and the bodies; the host-strip fallback and a device too small for
the sources (NativeError with LB2_E_CAPACITY) behave as in strip_tarball."""
import glob
import os
import shutil
import struct
import subprocess
import tarfile
import zipfile

import numpy as np
import pytest

import tar_archives as A
from test_gpu_strip_tarball import GOLDEN, LIMIT_CLASS, variant_tree, write_tgz
from test_layer_host import EPOCH_1980, compare, open_dirs, sorted_entries

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))


def literal(ctx, srcs, root, prefix, monkeypatch):
    """the passes zip_tarballs stands for, on disk: the entries of the sorted walk"""
    from lambdipy_b200.tarball import extract_tarball
    os.makedirs(root)
    dir_mtime = {}
    for s in srcs:
        extract_tarball(s, os.path.join(root, prefix), ctx=ctx)
        with tarfile.open(s, "r:gz") as t:
            for m in t.getmembers():
                if m.isdir():
                    dir_mtime[os.path.normpath(os.path.join(root, prefix, m.name))] = m.mtime
    modes = open_dirs(root)
    mtimes = {}
    for d, dirs, files in os.walk(root):
        for name in files:
            p = os.path.join(d, name)
            if not os.path.islink(p):
                mtimes[p] = os.stat(p).st_mtime_ns
    subprocess.run('find %s/ -name "*.so" | xargs strip' % root, shell=True, capture_output=True)
    for p, ns in mtimes.items():
        os.utime(p, ns=(ns, ns))                                           # strip -p
    for d, dirs, _ in os.walk(root, topdown=False):
        for name in dirs:
            p = os.path.join(d, name)
            if not os.path.islink(p):
                t = dir_mtime.get(os.path.normpath(p), EPOCH_1980)
                os.utime(p, (t, t))
    return sorted_entries(root, monkeypatch, modes)


def bodies(path):
    """{name: the member's DEFLATE body} of every file entry"""
    out = {}
    with zipfile.ZipFile(path) as zf, open(path, "rb") as f:
        for zi in zf.infolist():
            if zi.is_dir():
                continue
            f.seek(zi.header_offset)
            fh = struct.unpack(zipfile.structFileHeader, f.read(zipfile.sizeFileHeader))
            f.seek(fh[zipfile._FH_FILENAME_LENGTH] + fh[zipfile._FH_EXTRA_FIELD_LENGTH], 1)
            out[zi.filename] = f.read(zi.compress_size)
    return out


def check(ctx, srcs, tmp, monkeypatch, prefix="", levels=((None, None),), **kw):
    """zip_tarballs against the literal passes; bodies against zip_tree's at each (compresslevel, piece_bytes)"""
    from lambdipy_b200 import layer as L
    from lambdipy_b200 import zipfile_gpu as Z
    root = os.path.join(tmp, "tree")
    want = literal(ctx, srcs, root, prefix, monkeypatch)
    out = {}
    for level, piece in levels:
        extra = {} if piece is None else {"piece_bytes": piece}
        dst = os.path.join(tmp, "layer_%s_%s.zip" % (level, piece))
        st = L.zip_tarballs(srcs, dst, prefix=prefix, ctx=ctx, compresslevel=level, **extra, **kw)
        compare(dst, want)
        assert Z.testzip(dst, ctx=ctx) is None
        assert st["index"]["misses"] == 0 and st["entries"] == len(want) and st["zip_bytes"] == os.path.getsize(dst)
        got = bodies(dst)
        assert st["deflated_bytes"] == sum(len(b) for b in got.values())
        assert st["file_bytes"] == sum(zi.file_size for _, zi in want if not zi.is_dir())
        if st["fallback"] == 0:
            assert st["src_bytes"] == sum(os.path.getsize(s) for s in srcs)     # every body once, gzip headers not
            assert st["src_bytes"] - 512 * len(srcs) <= st["uploaded_bytes"] <= st["src_bytes"]
            assert st["downloaded_bytes"] == 16 * st["index"]["ranges"] + st["index"]["bytes"] + st["deflated_bytes"]
        ref = os.path.join(tmp, "ref.zip")
        Z.zip_tree(root, ref, ctx=ctx, compresslevel=level, **extra, **{k: v for k, v in kw.items() if k == "seek_table"})
        assert bodies(ref) == got
        os.unlink(ref)
        out[(level, piece)] = (st, dst)
    shutil.rmtree(root)
    return out


def test_variants_and_golden_two_sources(gpu_ctx, variants, tmp_path, monkeypatch):
    from lambdipy_b200 import layer as L
    root = variant_tree(str(tmp_path / "pkg"), variants)
    a = write_tgz(gpu_ctx, root, str(tmp_path / "a.tar.gz"), "tarfile")
    shutil.rmtree(root)
    groot = str(tmp_path / "golden")
    A.tree(groot, {os.path.basename(p)[:-7] + ".so": open(p, "rb").read()
                   for p in sorted(glob.glob(os.path.join(GOLDEN, "*.in.bin")))})
    b = write_tgz(gpu_ctx, groot, str(tmp_path / "b.tar.gz"), "gpu")
    shutil.rmtree(groot)
    runs = check(gpu_ctx, [a, b], str(tmp_path / "w"), monkeypatch,
                 levels=((None, None), (None, 1 << 20), (9, None)))
    st, dst = runs[(None, None)]
    assert st["gpu"] == st["selected"] > 10 and st["fallback"] == 0 and st["skipped"] == 1    # the directory x.so
    assert runs[(9, None)][0]["deflated_bytes"] <= st["deflated_bytes"]
    first = open(dst, "rb").read()
    L.zip_tarballs([a, b], dst, ctx=gpu_ctx)
    assert open(dst, "rb").read() == first                                                  # deterministic
    with zipfile.ZipFile(dst) as zf:
        for p in glob.glob(os.path.join(GOLDEN, "*.in.bin")):
            name = "golden/%s.so" % os.path.basename(p)[:-7]
            assert zf.read(name) == open(p[:-7] + ".gnu.bin", "rb").read()


def test_numpy_scipy_layer(gpu_ctx, tmp_path, monkeypatch):
    from lambdipy_b200 import zipfile_gpu as Z
    from lambdipy_b200.tarball import gzip_tarball
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    srcs = []
    for names, how in ((("numpy", "numpy.libs"), "tarfile"), (("scipy", "scipy.libs"), "gpu_seek")):
        paths = []
        for d in names:
            if os.path.exists(os.path.join(SITE, d)):
                shutil.copytree(os.path.join(SITE, d), tmp_path / "site" / d, symlinks=True)
                paths.append(str(tmp_path / "site" / d))
        dst = str(tmp_path / ("%s.tar.gz" % names[0]))
        if how == "tarfile":
            with tarfile.open(dst, "w:gz") as tar:
                for p in paths:
                    tar.add(p, arcname=os.path.basename(p))
        else:
            gzip_tarball(paths, dst, ctx=gpu_ctx, seek_table=True)
        srcs.append(dst)
    shutil.rmtree(tmp_path / "site")
    runs = check(gpu_ctx, srcs, str(tmp_path / "w"), monkeypatch, prefix="python/", seek_table=True)
    st, dst = runs[(None, None)]
    assert st["gpu"] + st["fallback"] == st["selected"] > 50 and st["members"] > 1000
    assert st["inflate"].get("seek_table", 0) > 0                        # the gzip_tarball source read from its table
    out = str(tmp_path / "back")
    ust = Z.extract_zip(dst, out, ctx=gpu_ctx)
    assert ust["seek_table"] > 0 and ust["seek_table_refused"] == 0
    with zipfile.ZipFile(dst) as zf:
        for zi in zf.infolist()[::50]:
            if not zi.is_dir():
                assert open(os.path.join(out, zi.filename), "rb").read() == zf.read(zi)
    print("numpy+scipy zip_tarballs:", {k: st[k] for k in ("members", "entries", "selected", "gpu", "fallback",
          "src_bytes", "zip_bytes", "kernel_ms")})


def test_fallback_non_elf_and_capacity(gpu_ctx, variants, tmp_path, monkeypatch):
    from lambdipy_b200 import _native as N
    from lambdipy_b200 import layer as L
    from lambdipy_b200.zipfile_gpu import StripFailed
    root = str(tmp_path / "pkg")
    A.tree(root, {"g.so": open(variants["c_g"], "rb").read(), "many.so": open(variants[LIMIT_CLASS], "rb").read(),
                  "text.so": b"this is not an ELF file\n" * 10})
    src = write_tgz(gpu_ctx, root, str(tmp_path / "s.tar.gz"), "gpu")
    shutil.rmtree(root)
    with pytest.raises(StripFailed, match="text.so"):
        L.zip_tarballs(src, str(tmp_path / "no.zip"), ctx=gpu_ctx)
    assert sorted(os.listdir(tmp_path)) == ["s.tar.gz"]
    runs = check(gpu_ctx, [src], str(tmp_path / "w"), monkeypatch, tolerate_non_elf=True)
    st, _ = runs[(None, None)]
    assert (st["gpu"], st["fallback"], st["skipped"]) == (1, 1, 1)
    assert st["uploaded_bytes"] > st["src_bytes"] and st["downloaded_bytes"] > os.path.getsize(variants[LIMIT_CLASS])
    real = gpu_ctx.dev_alloc

    def small_device(n):                       # a device without room for the sources' arena
        if n >= 1 << 20:
            raise N.NativeError(N.LB2_E_CUDA, "out of memory")
        return real(n)
    other = shutil.copy(src, str(tmp_path / "t.tar.gz"))
    monkeypatch.setattr(gpu_ctx, "dev_alloc", small_device)
    with pytest.raises(N.NativeError) as e:
        L.zip_tarballs([src, other], str(tmp_path / "no.zip"), ctx=gpu_ctx)
    monkeypatch.undo()
    assert e.value.code == N.LB2_E_CAPACITY
    assert sorted(os.listdir(tmp_path)) == ["s.tar.gz", "t.tar.gz", "w"]
