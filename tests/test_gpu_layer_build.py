"""GPU checks of zip_build (layer.py): tarballs and wheels to a Lambda zip, pip's target install and the clean-up
restated, shared objects inflated, stripped and deflated on the GPU.

Parity is with the passes run literally (test_layer_build_host.oracle): the tarballs extracted, the real pip 24 run
offline with --target, the build script's clean-up lines, the real `find -name "*.so" | xargs strip` (mtimes kept)
and the sorted walk: same names, order, modes, dates, sizes, CRC-32 and bytes.  The wheels are made here from the
installed numpy and scipy (the files their RECORD lists, packed with their .dist-info) and from the golden ELF files.
Also checked: both testzips, every selected file stripped on the GPU, the bytes uploaded, determinism, numpy as a
tarball mixed with scipy as a wheel, level 9, seek tables, the host-strip fallback and LB2_E_CAPACITY."""
import glob
import gzip
import importlib.metadata
import io
import os
import shutil
import stat
import subprocess
import tarfile
import zipfile

import numpy as np
import pytest

from test_gpu_strip_tarball import GOLDEN, LIMIT_CLASS
from test_layer_build_host import D1, oracle, whl

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))


def gnu_strip_tree(root):
    mtimes = {}
    for d, _, files in os.walk(root):
        for name in files:
            p = os.path.join(d, name)
            if not os.path.islink(p):
                mtimes[p] = os.stat(p).st_mtime_ns
    subprocess.run('find %s/ -name "*.so" | xargs strip' % root, shell=True, capture_output=True)
    for p, ns in mtimes.items():
        os.utime(p, ns=(ns, ns))                                               # strip -p


def installed_wheel(dist_name, out_dir):
    """a wheel of an installed distribution: the files its RECORD lists under site-packages, with their modes"""
    dist = importlib.metadata.distribution(dist_name)
    version = dist.version
    path = os.path.join(out_dir, "%s-%s-py3-none-any.whl" % (dist_name, version))
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for f in dist.files:
            rel = str(f)
            src = os.path.join(SITE, rel)
            if rel.startswith("..") or "__pycache__" in rel or not os.path.isfile(src) or os.path.islink(src):
                continue
            zi = zipfile.ZipInfo.from_file(src, rel)
            zi.compress_type = zipfile.ZIP_DEFLATED
            zi.date_time = D1
            zi.external_attr = (stat.S_IFREG | stat.S_IMODE(os.stat(src).st_mode)) << 16
            with open(src, "rb") as fh:
                zf.writestr(zi, fh.read())
    return path


def golden_wheel(out_dir, variants):
    files = [("elfpkg/%s.so" % os.path.basename(p)[:-7], open(p, "rb").read(), 0o755)
             for p in sorted(glob.glob(os.path.join(GOLDEN, "*.in.bin")))]
    files += [("elfpkg/v_%s.so" % k, open(v, "rb").read(), 0o755) for k, v in sorted(variants.items())
              if k != LIMIT_CLASS][:6]
    files += [("elfpkg/__init__.py", b"", 0o644), ("elfpkg/tests/test_x.py", b"x", 0o644),
              ("elfpkg-1.0.data/scripts/run", b"#!python\nimport elfpkg\n", 0o755)]
    return whl(os.path.join(out_dir, "elfpkg-1.0-py3-none-any.whl"), "elfpkg", "1.0", files, D1,
               entry_points="[console_scripts]\nelfpkg = elfpkg:main\n")


def selected_bodies(wheels, dst, prefix):
    """the compressed bodies of the wheel members that end up as selected files of dst"""
    with zipfile.ZipFile(dst) as zf:
        names = set(zf.namelist())
    total = 0
    for w in wheels:
        with zipfile.ZipFile(w) as zf:
            for n, zi in {zi.filename: zi for zi in zf.infolist()}.items():   # a repeated name: its last entry
                if n.endswith(".so") and prefix + n in names:
                    total += zi.compress_size
    return total


def check(ctx, tmp, monkeypatch, tars, tar_paths, wheels, prefix="", **kw):
    from lambdipy_b200 import layer as L
    from lambdipy_b200 import zipfile_gpu as Z
    from test_layer_host import compare
    want, _ = oracle(tars, wheels, tmp, monkeypatch, prefix, strip=gnu_strip_tree)
    dst = os.path.join(tmp, "layer.zip")
    st = L.zip_build(dst, tar_paths, wheels, prefix=prefix, ctx=ctx, **kw)
    compare(dst, want)
    assert Z.testzip(dst, ctx=ctx) is None
    assert st["entries"] == len(want) and st["zip_bytes"] == os.path.getsize(dst)
    shutil.rmtree(os.path.join(tmp, "tree"))
    shutil.rmtree(os.path.join(tmp, "work"))
    return st, dst


def test_golden_wheel_and_tarball(gpu_ctx, variants, tmp_path, monkeypatch):
    from lambdipy_b200 import layer as L
    w = golden_wheel(str(tmp_path), variants)
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        for k in sorted(variants)[:4]:
            if k != LIMIT_CLASS:
                tar.add(variants[k], arcname="tarpkg/%s.so" % k)
    tar_bytes = buf.getvalue()
    tgz = str(tmp_path / "tarpkg.tar.gz")
    with open(tgz, "wb") as f:
        f.write(gzip.compress(tar_bytes))
    for kw in ({}, {"compresslevel": 9}, {"seek_table": True, "piece_bytes": 1 << 20}):
        st, dst = check(gpu_ctx, str(tmp_path / "w"), monkeypatch, [tar_bytes], [tgz], [w], "python/", **kw)
        assert st["gpu"] == st["selected"] > 8 and st["fallback"] == 0 and st["generated_scripts"] == 1
        with zipfile.ZipFile(dst) as zf:
            made = sum(zf.getinfo("python/bin/" + n).file_size for n in ("elfpkg", "run"))
        rest = st["uploaded_bytes"] - selected_bodies([w], dst, "python/") - made   # the tarball, and padding
        assert os.path.getsize(tgz) - 512 <= rest <= os.path.getsize(tgz) + 32
    first = open(dst, "rb").read()
    L.zip_build(dst, [tgz], [w], prefix="python/", ctx=gpu_ctx, seek_table=True, piece_bytes=1 << 20)
    assert open(dst, "rb").read() == first                                                  # deterministic


def test_numpy_scipy_wheels_and_mixed(gpu_ctx, tmp_path, monkeypatch):
    from lambdipy_b200 import zipfile_gpu as Z
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    wdir = str(tmp_path / "wheels")
    os.makedirs(wdir)
    npw, spw = installed_wheel("numpy", wdir), installed_wheel("scipy", wdir)
    st, dst = check(gpu_ctx, str(tmp_path / "w1"), monkeypatch, [], [], [npw, spw], "python/")
    assert st["gpu"] + st["fallback"] == st["selected"] > 50 and st["copied"]["members"] > 1000
    bodies = selected_bodies([npw, spw], dst, "python/")
    if st["fallback"] == 0:
        assert bodies <= st["uploaded_bytes"] <= bodies + 16 * (st["generated_scripts"] + 1) + 4096
    assert zipfile.ZipFile(dst).testzip() is None
    print("numpy+scipy zip_build:", {k: st[k] for k in ("wheel_members", "entries", "selected", "gpu", "copied",
                                                         "removed", "zip_bytes", "kernel_ms")})
    # numpy as a tarball, scipy as a wheel, in one call
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        for d in ("numpy", "numpy.libs"):
            if os.path.exists(os.path.join(SITE, d)):
                tar.add(os.path.join(SITE, d), arcname=d)
    tgz = str(tmp_path / "numpy.tar.gz")
    with open(tgz, "wb") as f:
        f.write(gzip.compress(buf.getvalue(), compresslevel=1))
    st, dst = check(gpu_ctx, str(tmp_path / "w2"), monkeypatch, [buf.getvalue()], [tgz], [spw], "python/",
                    seek_table=True)
    assert st["gpu"] + st["fallback"] == st["selected"] > 50 and st["sources"] == 1 and st["wheels"] == 1
    ust = Z.extract_zip(dst, str(tmp_path / "back"), ctx=gpu_ctx)
    assert ust["seek_table"] > 0


def test_fallback_and_capacity(gpu_ctx, variants, tmp_path, monkeypatch):
    from lambdipy_b200 import _native as N
    from lambdipy_b200 import layer as L
    from lambdipy_b200.zipfile_gpu import StripFailed
    files = [("p/g.so", open(variants["c_g"], "rb").read(), 0o755),
             ("p/many.so", open(variants[LIMIT_CLASS], "rb").read(), 0o755),
             ("p/text.so", b"this is not an ELF file\n" * 10, 0o644)]
    w = whl(str(tmp_path / "p-1.0-py3-none-any.whl"), "p", "1.0", files, D1)
    with pytest.raises(StripFailed, match="text.so"):
        L.zip_build(str(tmp_path / "no.zip"), (), [w], ctx=gpu_ctx)
    assert not os.path.exists(tmp_path / "no.zip")
    st, _ = check(gpu_ctx, str(tmp_path / "w"), monkeypatch, [], [], [w], tolerate_non_elf=True)
    assert (st["gpu"], st["fallback"], st["skipped"]) == (1, 1, 1)
    real = gpu_ctx.dev_alloc

    def small_device(n):                       # a device without room for the tarballs' arena
        if n >= 1 << 20:
            raise N.NativeError(N.LB2_E_CUDA, "out of memory")
        return real(n)
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        tar.add(variants["c_g"], arcname="t/g.so")
        tar.add(variants[LIMIT_CLASS], arcname="t/many.so")
    tgz = [str(tmp_path / "a.tar.gz"), str(tmp_path / "b.tar.gz")]
    for t in tgz:
        with open(t, "wb") as f:
            f.write(gzip.compress(buf.getvalue()))
    monkeypatch.setattr(gpu_ctx, "dev_alloc", small_device)
    with pytest.raises(N.NativeError) as e:
        L.zip_build(str(tmp_path / "no.zip"), tgz, [w], ctx=gpu_ctx, tolerate_non_elf=True)
    monkeypatch.undo()
    assert e.value.code == N.LB2_E_CAPACITY
    assert not os.path.exists(tmp_path / "no.zip")
