"""CPU checks of zip_build's logic (lambdipy_b200.layer.build_with) with the stand-ins test_layer_host uses: zlib for
the readers and the encoder, a Python index and a fake `strip`, over a fake device memory.

The oracle is the contract run literally: the tarballs extracted into ./build (tree / prefix), the real pip 24 run
offline as `pip install --no-deps --no-index --target ./build W1.whl ...` on wheels this file writes with zipfile,
the build script's clean-up lines run by bash from the directory holding ./build, the fake strip on every `*.so`
(mtime kept, as `strip -p`), then the sorted walk of test_layer_host.  The documented deviations are applied to that
tree: a file pip wrote takes its wheel's date (every member of one test wheel has the same date, and the RECORD pip
writes says which wheel installed each path), a directory without a tarball member gets 1980-01-01.  As in
test_layer_host, directories are opened for the owner before the walk, so the oracle does not depend on who runs it;
pip's modes depend on the umask, which the oracle and zip_build read from the same process."""
import csv
import io
import os
import posixpath
import subprocess
import sys
import tarfile
import time
import zipfile

import pytest

from lambdipy_b200 import _native as N
from lambdipy_b200 import layer as L
from lambdipy_b200 import zipfile_gpu as Z
from test_layer_host import ArenaReader, EPOCH_1980, T0, compare, open_dirs, sorted_entries, tarb
from test_strip_tarball_host import PyIndex, gz
from test_strip_zip_host import DeviceZlibEncoder, FakeMemory, FakeStripper, ZlibDecoder, _pack, elf, fake_strip

D1, D2 = (2021, 3, 4, 5, 6, 8), (2022, 7, 8, 9, 10, 12)


class AnyBlockStripper(FakeStripper):
    """FakeStripper whose files may lie in several device blocks (a tar arena and the decoder's output), as
    GpuStripper reads every file at its own address"""

    def strip(self, refs):
        for b in self.mine:
            del self.mem.blocks[b]
        self.mine = []
        assert all(a % 16 == 0 for a, _ in refs)
        outs, status = [], []
        for ref in refs:
            d = self.mem.get(ref)
            refused = d[:5] == b"\x7fELF!"
            out = None if refused else fake_strip(d)
            status.append(N.ST_PLANNER_LIMIT if refused else N.ST_NOT_ELF if out is None else N.ST_OK)
            outs.append(out or b"")
        new = _pack(self.mem, outs, 256)
        if new:
            self.mine.append(new[0][0] >> 40 << 40)
        self.calls = getattr(self, "calls", 0) + 1
        return list(zip(status, new))


class SmallDecoder(ZlibDecoder):
    """a decoder with room for `room` members per run: DeviceTooSmall beyond it"""

    def __init__(self, mem, room):
        super().__init__(mem)
        self.room = room

    def run_device(self, n, members, tables=None):
        if len(members) > self.room:
            raise Z.DeviceTooSmall("stand-in")
        return super().run_device(n, members)


def whl(path, name, version, files, date, entry_points=None, wheel_version="1.0", info=None, methods=None):
    """a wheel: files [(name, bytes, mode)]; every member dated `date`"""
    info = info or "%s-%s.dist-info" % (name, version)
    meta = [(info + "/METADATA", b"Metadata-Version: 2.1\nName: %s\nVersion: %s\n" % (name.encode(), version.encode()),
             0o644),
            (info + "/WHEEL", b"Wheel-Version: %s\nGenerator: test\nRoot-Is-Purelib: true\nTag: py3-none-any\n"
             % wheel_version.encode(), 0o644)]
    if entry_points:
        meta.append((info + "/entry_points.txt", entry_points.encode(), 0o644))
    rows = [(n, "", "") for n, _, _ in files + meta] + [(info + "/RECORD", "", "")]
    buf = io.StringIO()
    csv.writer(buf).writerows(rows)
    with zipfile.ZipFile(path, "w") as zf:
        for n, data, mode in files + meta + [(info + "/RECORD", buf.getvalue().encode(), 0o644)]:
            zi = zipfile.ZipInfo(n, date)
            zi.external_attr = (0o100000 | mode) << 16
            zi.compress_type = (methods or {}).get(n, zipfile.ZIP_DEFLATED)
            zf.writestr(zi, data)
    return str(path)


def pip_install(target, wheels):
    env = dict(os.environ, PIP_CONFIG_FILE=os.devnull, PIP_NO_INPUT="1", PIP_DISABLE_PIP_VERSION_CHECK="1")
    r = subprocess.run([sys.executable, "-m", "pip", "install", "--no-deps", "--no-index", "--no-cache-dir",
                        "--target", target] + list(wheels), capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def cleanup_lines(work, keep_tests):
    from lambdipy_b200.project_build import _keep_pattern
    script = "\n".join(["set -e", "rm -rf ./build/*.egg-info", "rm -rf ./build/*.dist-info",
                        "find ./build/ -name __pycache__ | xargs rm -rf",
                        'find ./build/ -name tests | grep -v "%s" | xargs rm -rf' % _keep_pattern(keep_tests)])
    r = subprocess.run(["bash", "-c", script], cwd=work, capture_output=True)
    assert r.returncode == 0, r.stderr


def fake_strip_tree(root):
    """the fake strip on every `*.so` regular file under root, its mtime kept (strip -p)"""
    for d, dirs, files in os.walk(root):
        for name in files:
            p = os.path.join(d, name)
            if name.endswith(".so") and os.path.isfile(p) and not os.path.islink(p):
                st = os.stat(p)
                new = fake_strip(open(p, "rb").read())
                if new is not None:
                    with open(p, "r+b") as f:
                        f.write(new)
                        f.truncate()
                    os.utime(p, ns=(st.st_atime_ns, st.st_mtime_ns))


def oracle(tars, wheels, tmp, monkeypatch, prefix="", keep_tests=(), strip=fake_strip_tree):
    """the literal passes with the documented deviations applied: (entries, pip's output)"""
    work = os.path.join(tmp, "work")
    build = os.path.join(work, "build")
    os.makedirs(build)
    dir_mtime = {}
    for tar in tars:
        with tarfile.open(fileobj=io.BytesIO(tar)) as t:
            t.extractall(build, filter="fully_trusted")
            for m in t.getmembers():
                if m.isdir():
                    dir_mtime[os.path.normpath(os.path.join(build, m.name))] = m.mtime
    before = {os.path.join(d, f) for d, _, fs in os.walk(build) for f in fs}
    log = pip_install(build, wheels) if wheels else ""
    dates = {}                                          # installed path -> the date of the first wheel listing it
    for w in wheels:
        with zipfile.ZipFile(w) as zf:
            date = zf.infolist()[0].date_time
            info = [n for n in zf.namelist() if n.endswith(".dist-info/RECORD")][0].split("/")[0]
        rec = os.path.join(build, info, "RECORD")
        if not os.path.exists(rec):
            continue
        for row in csv.reader(open(rec)):
            p = posixpath.normpath(posixpath.join("lib/python", row[0]))
            p = p[len("lib/python/"):] if p.startswith("lib/python/") else p
            dates.setdefault(os.path.join(build, p), date)
    cleanup_lines(work, keep_tests)
    for d, _, fs in os.walk(build):
        for f in fs:
            p = os.path.join(d, f)
            if p not in before and p in dates and not os.path.islink(p):
                t = time.mktime(dates[p] + (0, 0, -1))
                os.utime(p, (t, t))
    root = os.path.join(tmp, "tree")
    if prefix:
        os.makedirs(os.path.dirname(os.path.join(root, prefix[:-1])))
        os.rename(build, os.path.join(root, prefix[:-1]))
        dir_mtime = {p.replace(build, os.path.join(root, prefix[:-1]), 1): t for p, t in dir_mtime.items()}
    else:
        os.rename(build, root)
        dir_mtime = {p.replace(build, root, 1): t for p, t in dir_mtime.items()}
    modes = open_dirs(root)
    strip(root)
    for d, dirs, _ in os.walk(root, topdown=False):
        for name in dirs:
            p = os.path.join(d, name)
            if not os.path.islink(p):
                t = dir_mtime.get(os.path.normpath(p), EPOCH_1980)
                os.utime(p, (t, t))
    return sorted_entries(root, monkeypatch, modes), log


def run(dst, tars=(), wheels=(), piece_bytes=1 << 20, room=None, **kw):
    mem = FakeMemory()
    dec = ZlibDecoder(mem) if room is None else SmallDecoder(mem, room)
    stripper = AnyBlockStripper(mem)
    st = L.build_with(str(dst), tars, wheels, ArenaReader(mem), PyIndex(mem), dec, stripper,
                      DeviceZlibEncoder(mem, piece_bytes), **kw)
    return st, stripper


def case(tmp, monkeypatch, tars, wheels, prefix="", keep_tests=(), **kw):
    srcs = [gz(os.path.join(tmp, "s%d.tar.gz" % i), t) for i, t in enumerate(tars)]
    dst = os.path.join(tmp, "out", "layer.zip")
    st, stripper = run(dst, srcs, wheels, prefix=prefix, keep_tests=keep_tests, **kw)
    want, log = oracle(tars, wheels, tmp, monkeypatch, prefix, keep_tests)
    compare(dst, want)
    assert os.listdir(os.path.join(tmp, "out")) == ["layer.zip"]
    assert st["entries"] == len(want) and st["zip_bytes"] == os.path.getsize(dst)
    return st, dst, log, stripper


def pkg_wheel(tmp, date=D1, name="pkgA", extra=()):
    files = [(name + "/__init__.py", b"from .core import *\n" * 30, 0o644),
             (name + "/core.so", elf(b"core of " + name.encode() * 200), 0o755),
             (name + "/tool.sh", b"#!/bin/sh\necho\n", 0o700),
             (name + "/tests/test_core.py", b"def test(): pass\n", 0o644),
             (name + "/sub/tests/data.bin", b"\0" * 300, 0o644),
             (name + "/sub/tests_extra.py", b"kept\n", 0o644),
             (name + "/__pycache__/core.cpython-312.pyc", b"pyc", 0o644),
             (name + "/vendored-1.0.dist-info/METADATA", b"below the top level: kept\n", 0o644),
             (name + ".libs/libgfortran-abc.so.5", elf(b"fortran " * 300), 0o755),
             (name + ".libs/libopen-x.so", elf(b"open " * 100), 0o644),
             ("extra.egg-info/PKG-INFO", b"gone\n", 0o644),
             ("top_module.py", b"print('top')\n", 0o644),
             (name + "-1.0.data/purelib/pure_mod.py", b"pure\n", 0o644),
             (name + "-1.0.data/platlib/plat_ext.so", elf(b"platlib"), 0o755),
             (name + "-1.0.data/headers/api.h", b"int api(void);\n", 0o644),
             (name + "-1.0.data/data/share/doc/readme.txt", b"data file\n", 0o644),
             (name + "-1.0.data/scripts/fixme", b"#!python -u\nimport sys\nprint(sys.argv)\n", 0o755),
             (name + "-1.0.data/scripts/fixme_plain", b"#!python\nprint(1)\n", 0o644),
             (name + "-1.0.data/scripts/shell.sh", b"#!/bin/sh\necho hi\n", 0o755),
             (name + "-1.0.data/scripts/" + name.lower() + "-cli", b"replaced by the entry point\n", 0o755),
             ] + list(extra)
    eps = "[console_scripts]\n%s-cli = %s.core:main\nother = %s:Cls.run [extra]\n\n[gui_scripts]\n%s-gui = %s:gui\n" \
        % (name.lower(), name, name, name.lower(), name)
    return whl(os.path.join(tmp, "%s-1.0-py3-none-any.whl" % name), name, "1.0", files, date, eps)


@pytest.mark.parametrize("prefix", ["", "python/"])
@pytest.mark.parametrize("keep_tests", [(), ("pkgA",)])
def test_tarball_and_wheels_against_pip(tmp_path, monkeypatch, prefix, keep_tests):
    a = pkg_wheel(str(tmp_path))
    shared = [("shared/common.py", b"same in both\n", 0o644)]
    b = whl(str(tmp_path / "pkg_b-2.0-cp312-cp312-manylinux_2_17_x86_64.whl"), "pkg_b", "2.0",
            [("pkg_b/__init__.py", b"b\n", 0o644), ("pkg_b/_b.cpython-312-x86_64-linux-gnu.so", elf(b"b" * 999), 0o755),
             ("pkg_b/tests/t.py", b"t\n", 0o644)] + shared, D2)
    a2 = whl(str(tmp_path / "pkg_c-1.0-py3-none-any.whl"), "pkg_c", "1.0", shared + [("c.py", b"c\n", 0o644)], D1)
    tar = tarb([("numpy/", ("dir",), 0o755, T0), ("numpy/core.so", elf(b"numpy " * 50), 0o755, T0 + 1),
                ("numpy/tests/", ("dir",), 0o755, T0), ("numpy/tests/t.py", b"t", 0o644, T0),
                ("numpy/__pycache__/x.pyc", b"x"), ("numpy-1.0.dist-info/RECORD", b"r"),
                ("pkgA/", ("dir",), 0o750, T0 + 5), ("pkgA/from_tarball.txt", b"the tarball holds pkgA", 0o644, T0)])
    st, dst, log, stripper = case(str(tmp_path), monkeypatch, [tar], [a, b, a2], prefix, keep_tests)
    assert "pkgA already exists" in log and st["skipped_items"] == ["pkgA"]          # pip skips the item whole
    assert st["wheels"] == 3 and st["generated_scripts"] == 3 and st["fallback"] == 0
    assert st["selected"] == st["gpu"] == 4 and stripper.calls == 1    # numpy, pkgA.libs, platlib, pkg_b: one batch
    assert st["removed"]["dist-info"] == 4 and st["removed"]["egg-info"] == 1 and st["removed"]["__pycache__"] == 1
    with zipfile.ZipFile(dst) as zf:
        names = zf.namelist()
        assert prefix + "bin/pkga-cli" in names and prefix + "pkgA/from_tarball.txt" in names
        assert zf.getinfo(prefix + "shared/common.py").date_time == D2                 # the first wheel listed
        fixed = zf.read(prefix + "bin/fixme")
        assert fixed.startswith(b"#!" + sys.executable.encode() + b"\n")
    assert st["copied"]["members"] > 5
    selected_bodies = sum(zi.compress_size for w in (a, b) for zi in zipfile.ZipFile(w).infolist()
                          if zi.filename.endswith(".so") and not zi.filename.startswith("pkgA/"))
    pad = st["uploaded_bytes"] - os.path.getsize(str(tmp_path / "s0.tar.gz")) - selected_bodies - host_made(dst, prefix)
    assert 0 <= pad < 16 * 5                # the five scripts made on the host go up in one 16-byte-aligned buffer


def host_made(dst, prefix):
    """bytes zip_build makes on the host: the fixed and generated scripts"""
    with zipfile.ZipFile(dst) as zf:
        return sum(zi.file_size for zi in zf.infolist() if zi.filename.startswith(prefix + "bin/") and
                   zi.filename.rsplit("/", 1)[1] in ("fixme", "fixme_plain", "pkga-cli", "other", "pkga-gui"))


def test_split_decoder_stored_members_and_pieces(tmp_path, monkeypatch):
    files = [("p/m%02d.so" % i, elf(b"%02d" % i * (i * 997 % 40_000)), 0o755) for i in range(12)] + \
        [("p/stored.txt", b"stored body " * 999, 0o644), ("p/big.bin", os.urandom(200_000), 0o644)]
    w = whl(str(tmp_path / "p-1.0-py3-none-any.whl"), "p", "1.0", files, D1,
            methods={"p/stored.txt": zipfile.ZIP_STORED, "p/m03.so": zipfile.ZIP_STORED})
    st, dst, _, stripper = case(str(tmp_path), monkeypatch, [], [w], piece_bytes=96 << 10)
    first = open(dst, "rb").read()
    assert st["gpu"] == 12 and st["copied"]["members"] == 1                  # big.bin; the stored member is decoded
    st2, _ = run(str(tmp_path / "split.zip"), (), [w], piece_bytes=96 << 10, room=3)
    assert open(str(tmp_path / "split.zip"), "rb").read() == first and st2["gpu"] == 12 and st2["fallback"] == 0


@pytest.mark.parametrize("bad", ["no_dist_info", "two_dist_info", "wheel_version", "leaves", "absolute", "method",
                                 "scheme_key", "name", "same_distribution", "overlap", "callable", "file_and_dir"])
def test_refusals(tmp_path, bad):
    t = str(tmp_path)
    ok = [("m/__init__.py", b"m\n", 0o644)]
    if bad == "no_dist_info":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok, D1, info="m-1.0.dist-info")]
        with zipfile.ZipFile(w[0]) as zf:
            items = [(zi, zf.read(zi)) for zi in zf.infolist() if ".dist-info" not in zi.filename]
        with zipfile.ZipFile(w[0], "w") as zf:
            for zi, data in items:
                zf.writestr(zi, data)
    elif bad == "two_dist_info":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok + [("n-1.0.dist-info/METADATA", b"", 0o644)], D1)]
    elif bad == "wheel_version":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok, D1, wheel_version="2.0")]
    elif bad == "leaves":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok + [("../evil.py", b"", 0o644)], D1)]
    elif bad == "absolute":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok + [("/etc/evil.py", b"", 0o644)], D1)]
    elif bad == "method":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok + [("m/x.so", b"x" * 100, 0o644)], D1,
                 methods={"m/x.so": zipfile.ZIP_BZIP2})]
    elif bad == "scheme_key":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok + [("m-1.0.data/lib/x", b"", 0o644)], D1)]
    elif bad == "name":
        w = [whl(t + "/m.whl", "m", "1.0", ok, D1)]
    elif bad == "same_distribution":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok, D1),
             whl(t + "/m-2.0-py3-none-any.whl", "m", "2.0", [("m2.py", b"", 0o644)], D1)]
    elif bad == "overlap":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok, D1),
             whl(t + "/n-1.0-py3-none-any.whl", "n", "1.0", [("m/__init__.py", b"other\n", 0o644)], D1)]
    elif bad == "callable":
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok, D1, entry_points="[console_scripts]\nm = m.main\n")]
    else:
        w = [whl(t + "/m-1.0-py3-none-any.whl", "m", "1.0", ok + [("m", b"a file", 0o644)], D1)]
    before = sorted(os.listdir(t))
    with pytest.raises(ValueError):
        run(t + "/o.zip", (), w)
    assert sorted(os.listdir(t)) == before


def test_identical_file_in_two_wheels_with_other_mode_is_refused(tmp_path):
    w = [whl(str(tmp_path / "m-1.0-py3-none-any.whl"), "m", "1.0", [("s/x.py", b"x", 0o644)], D1),
         whl(str(tmp_path / "n-1.0-py3-none-any.whl"), "n", "1.0", [("s/x.py", b"x", 0o755)], D1)]
    with pytest.raises(ValueError, match="different"):
        run(str(tmp_path / "o.zip"), (), w)


def test_clean_on_tarballs_only(tmp_path, monkeypatch):
    tar = tarb([("a/tests/t.py", b"t"), ("a/b/tests/u.py", b"u"), ("keep/tests/k.py", b"k"), ("x.dist-info/R", b"r"),
                (".hidden.dist-info/R", b"h"), ("a/__pycache__/c.pyc", b"c"), ("a/lib.so", elf(b"lib"))])
    st, dst, _, _ = case(str(tmp_path), monkeypatch, [tar], [], keep_tests=("keep",))
    assert st["removed"] == {"egg-info": 0, "dist-info": 1, "__pycache__": 1, "tests": 2, "entries": 8}
    with zipfile.ZipFile(dst) as zf:
        assert "keep/tests/k.py" in zf.namelist() and ".hidden.dist-info/R" in zf.namelist()


def test_cli(monkeypatch, capsys):
    seen = {}

    def fake(dst, tarballs, wheels, prefix="", keep_tests=(), compresslevel=None, seek_table=False):
        seen.update(dst=dst, tarballs=tarballs, wheels=wheels, prefix=prefix, keep=keep_tests, level=compresslevel,
                    seek=seek_table)
        return {"zip_bytes": 4e6, "src_bytes": 5e6, "entries": 12, "gpu": 3, "fallback": 1, "in_bytes": 5e6,
                "out_bytes": 1e6, "copied": {"members": 7}, "removed": {"entries": 2}}
    monkeypatch.setattr(L, "zip_build", fake)
    assert L.main(["l.zip", "--wheel", "a.whl", "--wheel", "b.whl", "--prefix", "python/", "--keep-tests", "x",
                   "--seek-table"]) == 0
    assert seen == {"dst": "l.zip", "tarballs": [], "wheels": ["a.whl", "b.whl"], "prefix": "python/", "keep": ["x"],
                    "level": None, "seek": True}
    out = capsys.readouterr().out.strip().splitlines()
    assert len(out) == 1 and "7 bodies copied" in out[0] and "4 shared objects stripped (1 via host strip)" in out[0]
    assert L.main(["l.zip", "t.tar.gz", "--clean", "--level", "9"]) == 0
    assert seen["tarballs"] == ["t.tar.gz"] and seen["wheels"] == [] and seen["level"] == 9
    called = {}
    monkeypatch.setattr(L, "zip_tarballs", lambda *a, **k: called.setdefault("zip_tarballs", (a, k)) and
                        {"zip_bytes": 1, "src_bytes": 1, "entries": 1, "gpu": 0, "fallback": 0, "in_bytes": 0,
                         "out_bytes": 0})
    assert L.main(["l.zip", "t.tar.gz"]) == 0 and "zip_tarballs" in called              # no new flag: unchanged
    for bad in (["l.zip"], ["l.zip", "t.tar.gz", "--keep-tests", "x"]):
        with pytest.raises(SystemExit):
            L.main(bad)
    import lambdipy_b200
    assert lambdipy_b200.zip_build is fake
