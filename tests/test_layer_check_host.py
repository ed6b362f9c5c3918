"""CPU checks of the check that zip_build and zip_tarballs run before they write (build_with / zip_with with check=...),
behind the stand-ins of test_layer_build_host and test_layer_host (zlib for the readers and the encoder, a Python
index, a fake `strip`, a fake device memory), the emulator of the dynamic-section parse (deps_lib) and the emulator
of the symbol index and lookup (syms_lib).

The oracle is check_with on the zip that was written, behind the same stand-ins: stats["check"] must equal its report,
the whole of it apart from the engine timings and bus bytes in stats, which the writer's check counts differently (it
reuses the bytes the build holds on the device).  A check with problems raises CheckFailed with the report check_with
gives for the zip written without the check, and leaves dst as it was.

The objects are linked by gcc with -s and carry the fake strip's marker at their end, so the fake strip gives back the
linked object; the symbol fixtures are test_symbols_host's."""
import os
import subprocess
import zipfile

import pytest

import syms_lib as S
from lambdipy_b200 import _native as N
from lambdipy_b200 import deps
from lambdipy_b200 import layer as L
from test_deps_host import EmuParser, TableZlibDecoder
from test_layer_build_host import D1, AnyBlockStripper, SmallDecoder, whl
from test_layer_host import ArenaReader, tarb
from test_strip_tarball_host import PyIndex, gz
from test_strip_zip_host import MARK, DeviceZlibEncoder, FakeMemory, ZlibDecoder
from test_symbols_host import emu, fx  # noqa: F401  (fixtures)

STAT_KEYS = ("members", "roots", "objects", "rounds", "references", "lookups", "symbols_skipped")
HOST_STRIP = b"strip me on the host"


class HostOnlyStripper(AnyBlockStripper):
    """AnyBlockStripper that refuses the objects holding HOST_STRIP, which the host strip then takes"""

    def strip(self, refs):
        out = super().strip(refs)
        return [(N.ST_PLANNER_LIMIT if HOST_STRIP in self.mem.get(r) else st, new) for r, (st, new) in zip(refs, out)]


def _cc(d, name, code, *args):
    src = os.path.join(d, name + ".c")
    with open(src, "w") as f:
        f.write(code)
    p = os.path.join(d, name)
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-s", "-o", p, src, "-L" + d] + list(args), check=True,
                   capture_output=True)
    return p


def unstripped(path):
    """the linked object with the fake strip's marker and a debug tail after it"""
    data = open(path, "rb").read()
    assert MARK not in data
    return data + MARK + b"debug info " * 40


@pytest.fixture(scope="module")
def objs(tmp_path_factory):
    """{name: bytes}: libgf.so.5; libx.so.1 (needs libgf.so.5, DT_RPATH $ORIGIN); _ext.so (needs libx.so.1, DT_RPATH
    $ORIGIN/../pkg.libs); _core.so (needs libgf.so.5, DT_RPATH $ORIGIN/../w.libs); _gone.so
    (needs libgone.so.1, absent); _host.so (stripped on the host only)"""
    d = str(tmp_path_factory.mktemp("layer_check"))
    out = {}
    out["libgf.so.5"] = _cc(d, "libgf.so.5", "int gf(void) { return 5; }\n", "-Wl,-soname,libgf.so.5")
    out["libx.so.1"] = _cc(d, "libx.so.1", "int gf(void);\nint xf(void) { return gf(); }\n", "-l:libgf.so.5",
                           "-Wl,-soname,libx.so.1", "-Wl,--disable-new-dtags,-rpath,$ORIGIN")
    out["_ext.so"] = _cc(d, "_ext.so", "int xf(void);\nint e(void) { return xf(); }\n", "-l:libx.so.1",
                         "-Wl,--disable-new-dtags,-rpath,$ORIGIN/../pkg.libs")
    out["_core.so"] = _cc(d, "_core.so", "int gf(void);\nint c(void) { return gf(); }\n", "-l:libgf.so.5",
                          "-Wl,--disable-new-dtags,-rpath,$ORIGIN/../w.libs")
    _cc(d, "libgone.so.1", "int gone(void) { return 0; }\n", "-Wl,-soname,libgone.so.1")
    out["_gone.so"] = _cc(d, "_gone.so", "int gone(void);\nint g(void) { return gone(); }\n", "-l:libgone.so.1")
    out["_host.so"] = _cc(d, "_host.so", "const char *h(void) { return \"%s\"; }\n" % HOST_STRIP.decode())
    return {k: unstripped(p) for k, p in out.items()}


def ext_tar(objs, extra=()):
    """pkg/_ext.so, and under pkg.libs libx.so.1 with the link libx.so -> libx.so.1, and libgf.so.5"""
    return tarb([("pkg/", ("dir",), 0o755), ("pkg/_ext.so", objs["_ext.so"], 0o755),
                 ("pkg.libs/", ("dir",), 0o755), ("pkg.libs/libx.so.1", objs["libx.so.1"], 0o755),
                 ("pkg.libs/libx.so", ("sym", "libx.so.1")), ("pkg.libs/libgf.so.5", objs["libgf.so.5"], 0o755),
                 ("pkg/__init__.py", b"from ._ext import *\n")] + list(extra))


def core_wheel(tmp, objs, extra=(), name="w", methods=None):
    """a wheel whose root w/_core.so needs w.libs/libgf.so.5, a member only round 2 reaches"""
    return whl(os.path.join(tmp, "%s-1.0-cp312-cp312-manylinux_2_17_x86_64.whl" % name), name, "1.0",
               [(name + "/__init__.py", b"from ._core import *\n", 0o644), (name + "/_core.so", objs["_core.so"], 0o755),
                (name + ".libs/libgf.so.5", objs["libgf.so.5"], 0o755)] + list(extra), D1, methods=methods)


class Engines:
    """the stand-ins of one run over one fake device memory"""

    def __init__(self, emu, check, room=None, stripper=AnyBlockStripper):
        self.mem = mem = FakeMemory()
        self.dec = ZlibDecoder(mem) if room is None else SmallDecoder(mem, room)
        self.parser = EmuParser(mem, emu)
        self.resolver = S.EmuResolver(mem) if check and check.get("symbols") else None
        self.stripper = stripper(mem)
        self.kw = dict(check=check, parser=self.parser if check is not None else None, resolver=self.resolver)

    def build(self, dst, tars=(), wheels=(), **kw):
        return L.build_with(str(dst), tars, wheels, ArenaReader(self.mem), PyIndex(self.mem), self.dec, self.stripper,
                            DeviceZlibEncoder(self.mem), **self.kw, **kw)

    def zip(self, dst, tars, **kw):
        return L.zip_with(tars, str(dst), ArenaReader(self.mem), PyIndex(self.mem), self.stripper,
                          DeviceZlibEncoder(self.mem), **self.kw, **kw)


def check_dst(dst, emu, check):
    mem = FakeMemory()
    return deps.check_with(dst, TableZlibDecoder(mem), EmuParser(mem, emu), **check,
                           **({"resolver": S.EmuResolver(mem)} if check.get("symbols") else {}))


def same(got, want):
    strip_stats = lambda r: {k: v for k, v in r.items() if k != "stats"}  # noqa: E731
    assert strip_stats(got) == strip_stats(want)
    assert {k: got["stats"].get(k) for k in STAT_KEYS} == {k: want["stats"].get(k) for k in STAT_KEYS}


def layer(tmp, emu, check, tars=(), wheels=(), how="build", room=None, stripper=AnyBlockStripper, **kw):
    """write the zip with and without the check: (stats with the check, the zip's path, the engines); the two zips
    must be byte for byte the same and the report check_with's on them"""
    srcs = [gz(os.path.join(tmp, "s%d.tar.gz" % i), t) for i, t in enumerate(tars)]
    plain = os.path.join(tmp, "plain.zip")
    dst = os.path.join(tmp, "out", "layer.zip")
    e0, e = Engines(emu, None, room, stripper), Engines(emu, check, room, stripper)
    if how == "build":
        st0 = e0.build(plain, srcs, wheels, **kw)
        st = e.build(dst, srcs, wheels, **kw)
    else:
        st0 = e0.zip(plain, srcs, **kw)
        st = e.zip(dst, srcs, **kw)
    assert "check" not in st0 and open(dst, "rb").read() == open(plain, "rb").read()
    bus = ("check", "uploaded_bytes", "downloaded_bytes")   # a member left in the decoder's output goes via the host
    assert {k: v for k, v in st.items() if k not in bus} == {k: v for k, v in st0.items() if k not in bus}
    assert os.listdir(os.path.dirname(dst)) == ["layer.zip"]
    same(st["check"], check_dst(dst, emu, check))
    c = st["check"]["stats"]
    assert c["roots_reused"] == c["roots"] > 0
    return st, dst, e


@pytest.mark.parametrize("how", ["build", "zip"])
@pytest.mark.parametrize("prefix,mount", [("", "/var/task"), ("python/", "/opt")])
def test_tarball_links_and_origin_rpath(tmp_path, emu, objs, how, prefix, mount):
    st, dst, e = layer(str(tmp_path), emu, {"mount": mount}, [ext_tar(objs)], how=how, prefix=prefix)
    rep = st["check"]
    top = mount + "/" + prefix
    base = top + "pkg.libs/"
    # libx.so and libx.so.1 are two entries with the same bytes: two objects, as in the zip
    assert {base + "libx.so", base + "libx.so.1", base + "libgf.so.5"} <= set(rep["objects"])
    assert rep["closures"][top + "pkg/_ext.so"] == [top + "pkg/_ext.so", base + "libx.so.1", base + "libgf.so.5"]
    assert rep["stats"]["rounds"] == 2 and rep["stats"]["roots"] == 2 and rep["problems"] == []
    assert rep["stats"]["bytes_up"] == 0 and e.parser.uploaded == 0        # every byte was on the device already


@pytest.mark.parametrize("prefix,mount", [("", "/var/task"), ("python/", "/opt")])
def test_wheel_member_reached_in_round_two(tmp_path, emu, objs, prefix, mount):
    # a stored member is decoded with the roots and must outlive the decoder's round-two run
    w = core_wheel(str(tmp_path), objs, [("w/data.bin", b"stored " * 500, 0o644)],
                   methods={"w/data.bin": zipfile.ZIP_STORED})
    st, dst, e = layer(str(tmp_path), emu, {"mount": mount}, wheels=[w], prefix=prefix)
    rep = st["check"]
    top = mount + "/" + prefix
    assert rep["closures"][top + "w/_core.so"] == [top + "w/_core.so", top + "w.libs/libgf.so.5"]
    assert rep["stats"]["rounds"] == 2 and st["copied"]["members"] >= 1
    body = zipfile.ZipFile(w).getinfo("w.libs/libgf.so.5").compress_size
    assert rep["stats"]["bytes_up"] == body                                 # the round-two body, and no root


def test_tarball_mixed_with_wheels_split_decoder(tmp_path, emu, objs):
    w = core_wheel(str(tmp_path), objs)
    w2 = core_wheel(str(tmp_path), objs, name="v")
    want = None
    for room in (None, 1):
        d = tmp_path / ("room%s" % room)
        d.mkdir()
        st, _, _ = layer(str(d), emu, {"mount": "/opt"}, [ext_tar(objs)], [w, w2], prefix="python/", room=room)
        rep = st["check"]
        assert rep["problems"] == [] and rep["stats"]["roots"] == 4
        if want is None:
            want = rep
        same(rep, want)


def test_host_fallback_root(tmp_path, emu, objs):
    tar = ext_tar(objs, [("pkg/_host.so", objs["_host.so"], 0o755)])
    w = core_wheel(str(tmp_path), objs, [("w/_host2.so", objs["_host.so"], 0o755)])
    st, _, _ = layer(str(tmp_path), emu, {}, [tar], [w], stripper=HostOnlyStripper)
    assert st["fallback"] == 2 and st["check"]["objects"]["/var/task/pkg/_host.so"]["status"] == "ok"


def test_host_made_script_named_so_under_tolerate_non_elf(tmp_path, emu, objs):
    w = core_wheel(str(tmp_path), objs, [("w-1.0.data/scripts/tool.so", b"#!python\nprint(1)\n", 0o755),
                                         ("w/stored.so", b"not an object", 0o644)])
    plain = str(tmp_path / "plain.zip")
    st0 = Engines(emu, None).build(plain, (), [w], tolerate_non_elf=True)
    assert st0["skipped"] == 2
    dst = tmp_path / "out.zip"
    with pytest.raises(deps.CheckFailed) as e:                             # what check_zip says of such a zip
        Engines(emu, {}).build(dst, (), [w], tolerate_non_elf=True)
    same(e.value.report, check_dst(plain, emu, {}))
    assert {p["object"] for p in e.value.report["problems"]} == {"/var/task/bin/tool.so", "/var/task/w/stored.so"}
    assert e.value.report["stats"]["roots_reused"] == e.value.report["stats"]["roots"] == 3
    assert not dst.exists()


def test_symbols(tmp_path, emu, fx):
    ok = {"symbols": True, "ld_library_path": "/var/task/lib"}
    files = {"pkg/user.so": fx["user"], "lib/libdef.so": fx["def_gnu"], "pkg/kinds_user.so": fx["kinds_user"],
             "lib/libkinds.so": fx["kinds"], "lib/libuniq.so": fx["uniq"], "pkg/z_user.so": fx["z_user"]}
    tar = tarb([(n, open(p, "rb").read(), 0o755) for n, p in files.items()])
    st, _, _ = layer(str(tmp_path), emu, ok, [tar])
    rep = st["check"]
    assert rep["problems"] == [] and rep["symbols"]["/var/task/pkg/user.so"]["in_zip"] == 2
    assert rep["stats"]["references"] > 0 and rep["stats"]["lookups"] > 0


@pytest.mark.parametrize("what", ["need", "symbol"])
def test_problems_raise_and_leave_dst(tmp_path, emu, objs, fx, what):
    t = str(tmp_path)
    if what == "need":
        check, tar = {}, ext_tar(objs, [("pkg/_gone.so", objs["_gone.so"], 0o755)])
    else:
        check = {"symbols": True, "ld_library_path": "/var/task/lib"}
        tar = tarb([("pkg/user.so", open(fx["user"], "rb").read(), 0o755),
                    ("lib/libdef.so", open(fx["def_noB"], "rb").read(), 0o755)])
    src = gz(os.path.join(t, "s.tar.gz"), tar)
    plain = os.path.join(t, "plain.zip")
    Engines(emu, None).build(plain, [src])
    want = check_dst(plain, emu, check)
    out = os.path.join(t, "out")
    os.makedirs(out)
    dst = os.path.join(out, "layer.zip")
    with open(dst, "wb") as f:
        f.write(b"the previous layer")
    for how in ("build", "zip"):
        e = Engines(emu, check)
        with pytest.raises(deps.CheckFailed) as got:
            e.build(dst, [src]) if how == "build" else e.zip(dst, [src])
        same(got.value.report, want)
        assert open(dst, "rb").read() == b"the previous layer" and os.listdir(out) == ["layer.zip"]
    kinds = {p["kind"] for p in want["problems"]}
    assert kinds == ({"missing"} if what == "need" else {"symbol"})
    detail = want["problems"][0]["detail"]
    assert ("libgone.so.1" in detail) if what == "need" else detail.startswith("b_fn: no definition")


@pytest.mark.parametrize("check", [{"mount": "/opt", "symbol": True}, {"arch": "sparc"},
                                   {"max_versions": {"GLIBC": "new"}}, ["mount"]])
def test_refused_check_raises_before_anything_is_read(tmp_path, emu, check):
    class Unread:
        def __getattr__(self, name):
            raise AssertionError("%s used before the check was refused" % name)
    missing = str(tmp_path / "absent.tar.gz"), str(tmp_path / "absent-1.0-py3-none-any.whl")
    for call in (lambda: L.build_with(str(tmp_path / "o.zip"), [missing[0]], [missing[1]], Unread(), Unread(), Unread(),
                                      Unread(), Unread(), check=check, parser=Unread()),
                 lambda: L.zip_with([missing[0]], str(tmp_path / "o.zip"), Unread(), Unread(), Unread(), Unread(),
                                    check=check, parser=Unread())):
        with pytest.raises(ValueError):
            call()
    with pytest.raises(ValueError):
        L.zip_build(str(tmp_path / "o.zip"), wheels=[missing[1]], check=check)
    assert sorted(os.listdir(str(tmp_path))) == []


def test_cli_exit_codes(monkeypatch, capsys):
    seen = {}
    report = {"arch": "x86_64", "mount": "/opt", "max_versions": {}, "provided_used": {}, "problems": [], "notes": [],
              "stats": {"objects": 3, "roots": 2, "rounds": 2}}
    st = {"zip_bytes": 4e6, "src_bytes": 5e6, "entries": 12, "gpu": 3, "fallback": 0, "in_bytes": 5e6,
          "out_bytes": 1e6, "copied": {"members": 7}, "removed": {"entries": 2}, "check": report}

    def fake(dst, tarballs, wheels, prefix="", keep_tests=(), compresslevel=None, seek_table=False, check=None):
        seen.update(check=check)
        if check["arch"] == "arm64":
            raise deps.CheckFailed(dict(report, problems=[{"object": "/opt/python/a.so", "kind": "arch",
                                                          "detail": "e_machine 62, not arm64 (183)"}]))
        return st
    monkeypatch.setattr(L, "zip_build", fake)
    base = ["l.zip", "--wheel", "a.whl", "--prefix", "python/", "--check", "--mount", "/opt"]
    assert L.main(base + ["--symbols", "--interpreter", "/usr/bin/python3", "--max-version", "GLIBC_2.26"]) == 0
    assert seen["check"] == {"mount": "/opt", "arch": "x86_64", "provided": deps.DEFAULT_PROVIDED,
                             "max_versions": {"GLIBC": "2.26"}, "ld_library_path": deps.LAMBDA_LD_LIBRARY_PATH,
                             "symbols": True, "interpreter": ["/usr/bin/python3"], "runtime_libs": []}
    out = capsys.readouterr().out.splitlines()
    assert out[0].startswith("Layer zip: l.zip") and out[1] == deps.summary(report).splitlines()[0]
    assert L.main(base + ["--arch", "arm64"]) == 1
    out = capsys.readouterr().out
    assert "l.zip not written" in out and "problem: /opt/python/a.so: arch" in out
    assert L.main(base + ["--max-version", "GLIBC"]) == 2                  # refused by the check's own rule
    monkeypatch.setattr(L, "zip_build", lambda *a, **k: (_ for _ in ()).throw(ValueError("a bad wheel")))
    assert L.main(base) == 2 and "a bad wheel" in capsys.readouterr().err
    monkeypatch.setattr(L, "zip_tarballs", lambda srcs, dst, **k: seen.update(tar_check=k.get("check")) or st)
    assert L.main(["l.zip", "t.tar.gz", "--check", "--provided", "libc.so.6"]) == 0
    assert seen["tar_check"]["provided"] == frozenset(["libc.so.6"])
    with pytest.raises(SystemExit) as e:                                    # a check option without --check
        L.main(["l.zip", "t.tar.gz", "--symbols"])
    assert e.value.code == 2
