"""CPU checks of check_zip's loader model (lambdipy_b200.deps.check_with) behind zlib and the g++ build of the product's
parse (tests/emu/deps_emu.cpp over elf_deps.cuh), with the real glibc loader as the oracle: each fixture zip is
extracted under a temporary directory used as the mount, `ld_library_path` is mapped onto it, and
`ld-linux-x86-64.so.2 --list ROOT` must resolve every name to the same member, or to "not found", as the model does
(`provided` being what the loader found outside the tree).

Covered: RPATH vs RUNPATH precedence, the RPATH loader chain (and RUNPATH not being inherited), $ORIGIN, /opt/lib and
/var/task/lib through LD_LIBRARY_PATH, both mounts, symlink entries, SONAME matches, missing libraries, arch
mismatches, VERDEF misses, weak needs, ceilings, the numpy + scipy layer in three rounds, and the command's exit
codes."""
import os
import posixpath
import re
import shutil
import stat
import subprocess
import zipfile

import pytest

import deps_lib as D
import elf_fixtures as F
from lambdipy_b200 import _native as N
from lambdipy_b200 import deps
from test_strip_zip_host import FakeMemory, ZlibDecoder

LD_SO = "/lib64/ld-linux-x86-64.so.2"


class EmuParser:
    """GpuElfParser's interface over the emulator and the fake device memory"""

    def __init__(self, mem, emu, edit=None):
        self.mem, self.emu, self.edit = mem, emu, edit
        self.uploaded = self.downloaded = 0
        self.batches = []

    def parse(self, refs):
        blobs = [self.mem.get(r) for r in refs]
        self.batches.append(len(refs))
        out = self.emu.parse(blobs)
        return [self.edit(o) for o in out] if self.edit else out

    def upload(self, data):
        self.uploaded += len(data)
        return self.mem.put(data), len(data)

    def stats(self):
        return {"kernel_ms": 0.0}


@pytest.fixture(scope="module")
def emu():
    return D.Emu()


class TableZlibDecoder(ZlibDecoder):
    """zlib reads a member with a seek table as any other"""

    def run_device(self, n, members, tables=None):
        return super().run_device(n, members)


def check(zip_path, emu, edit=None, **kw):
    mem = FakeMemory()
    return deps.check_with(zip_path, TableZlibDecoder(mem), EmuParser(mem, emu, edit), **kw)


def cc(out, src, *args):
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-o", out, src] + list(args), check=True, capture_output=True)
    return out


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    """small libraries: liba (soname liba.so.1), libv (versions V1 V2), libv1only (V1 only, soname libv.so), libmid
    (needs libdeep.so, no search path of its own), libdeep, and an aarch64-tagged copy of liba"""
    d = str(tmp_path_factory.mktemp("deps_libs"))
    def src(name, text):
        p = os.path.join(d, name)
        with open(p, "w") as f:
            f.write(text)
        return p
    a, v = src("a.c", D.LIB_A), src("v.c", D.LIB_V)
    vs, v1 = src("v.map", D.VSCRIPT), src("v1.map", "V1 { global: v1; local: *; };\nV2 { global: v2; } V1;\n")
    out = {"liba": cc(os.path.join(d, "liba.so.1.0"), a, "-Wl,-soname,liba.so.1"),
           "libv": cc(os.path.join(d, "libv.so"), v, "-Wl,--version-script=" + vs, "-Wl,-soname,libv.so"),
           "libdeep": cc(os.path.join(d, "libdeep.so"), src("deep.c", "int deep(void) { return 3; }\n"))}
    os.makedirs(os.path.join(d, "v1"))
    out["libv1only"] = cc(os.path.join(d, "v1", "libv.so"), src("v1.c", "int v1(void) { return 1; }\n"),
                          "-Wl,--version-script=" + src("only.map", "V1 { global: v1; local: *; };\n"), "-Wl,-soname,libv.so")
    out["libmid"] = cc(os.path.join(d, "libmid.so"), src("mid.c", "int deep(void);\nint mid(void) { return deep(); }\n"),
                       "-L" + d, "-ldeep")
    user = src("user.c", D.USER)
    shutil.copy(out["liba"], os.path.join(d, "liba.so"))

    def user_lib(name, *args):
        return cc(os.path.join(d, name), user, "-L" + d, *args, "-lv", "-la")
    out["u_rpath"] = user_lib("u_rpath.so", "-Wl,--disable-new-dtags,-rpath,$ORIGIN/../lib")
    out["u_runpath"] = user_lib("u_runpath.so", "-Wl,--enable-new-dtags,-rpath,$ORIGIN/../lib")
    out["u_plain"] = user_lib("u_plain.so")
    mid_user = src("mu.c", "int mid(void);\nint mu(void) { return mid(); }\n")
    for dt, flag in (("rpath", "--disable-new-dtags"), ("runpath", "--enable-new-dtags")):
        out["chain_" + dt] = cc(os.path.join(d, "chain_%s.so" % dt), mid_user, "-L" + d, "-lmid",
                                "-Wl,%s,-rpath,$ORIGIN/../lib:$ORIGIN/../deep" % flag)
    arm = bytearray(open(out["liba"], "rb").read())
    arm[18:20] = (183).to_bytes(2, "little")
    out["liba_arm"] = os.path.join(d, "liba_arm.so")
    with open(out["liba_arm"], "wb") as f:
        f.write(arm)
    return out


def make_zip(path, entries, compression=zipfile.ZIP_DEFLATED):
    """entries: {name: file path | ("link", target)}"""
    with zipfile.ZipFile(path, "w", compression) as zf:
        for name, what in entries.items():
            if isinstance(what, tuple):
                zi = zipfile.ZipInfo(name)
                zi.external_attr = (stat.S_IFLNK | 0o777) << 16
                zf.writestr(zi, what[1])
            else:
                zf.write(what, name)
    return path


def extract(zip_path, root):
    """unzip with symlink entries made symlinks"""
    with zipfile.ZipFile(zip_path) as zf:
        for zi in zf.infolist():
            p = os.path.join(root, zi.filename)
            os.makedirs(os.path.dirname(p), exist_ok=True)
            if (zi.external_attr >> 16) & 0o170000 == stat.S_IFLNK:
                os.symlink(zf.read(zi).decode(), p)
            elif not zi.is_dir():
                with open(p, "wb") as f:
                    f.write(zf.read(zi))


def loader_list(root_file, library_path):
    """({name: resolved path (normalised) or None}, whether the loader stopped) from the real loader's --list"""
    r = subprocess.run([LD_SO, "--library-path", library_path, "--list", root_file], capture_output=True, text=True)
    m = re.search(r"error while loading shared libraries: (\S+): cannot open shared object file", r.stderr)
    if m:  # a need below the root's own resolves nowhere: the loader stops there and lists nothing
        return {m.group(1): None}, True
    out = {}
    for line in r.stdout.splitlines():
        m = re.match(r"^\s+(\S+) => (not found|(\S+) \(0x[0-9a-f]+\))$", line)
        if m:
            out[m.group(1)] = None if m.group(2) == "not found" else os.path.normpath(m.group(3))
    return out, False


def oracle_compare(tmp_path, zip_path, emu, mount, ld_dirs, roots=None):
    """the model against the real loader on every root (or the given ones); returns the report"""
    tree = str(tmp_path / "tree")
    base = tree + mount
    extract(zip_path, base)
    lib_path = ":".join(tree + d for d in ld_dirs)
    got = {}
    with zipfile.ZipFile(zip_path) as zf:
        root_names = [zi.filename for zi in zf.infolist() if deps.Z.selected_for_strip(zi)]
    for name in root_names if roots is None else roots:
        got[name] = loader_list(os.path.join(base, name), lib_path)
    provided = {n for res, _ in got.values() for n, p in res.items() if p is not None and not p.startswith(tree + "/")}
    provided.add(os.path.basename(LD_SO))  # --list prints the loader itself without "=>"
    report = check(zip_path, emu, mount=mount, provided=provided, ld_library_path=":".join(ld_dirs))
    for name, (res, stopped) in got.items():
        model = model_resolutions(report, posixpath.join(mount, name))
        for need, p in res.items():
            want = None if p is None else ("provided" if not p.startswith(tree + "/") else p[len(tree):])
            if need in model or want != "provided":  # a provided library's own needs are not modelled
                assert model.get(need) == want, (name, need, model.get(need), want)
        assert stopped or set(model) - {os.path.basename(LD_SO)} <= set(res), (name, set(model) ^ set(res))
    return report


def model_resolutions(report, root):
    """{name: mounted path, "provided" or None} of the root's load, as --list prints it (first resolution)"""
    out = {}
    for r in report["resolved"][root]:
        out.setdefault(r["name"], {"missing": None, "provided": "provided"}.get(r["how"], r["path"]))
    return out


def test_rpath_runpath_origin_and_symlinks(tmp_path, emu, libs):
    z = make_zip(str(tmp_path / "b.zip"), {
        "pkg/u_rpath.so": libs["u_rpath"], "pkg/u_runpath.so": libs["u_runpath"],
        "lib/liba.so.1.0": libs["liba"], "lib/liba.so.1": ("link", "liba.so.1.0"), "lib/libv.so": libs["libv"]})
    rep = oracle_compare(tmp_path, z, emu, "/var/task", ["/nonexistent"])
    assert rep["problems"] == []
    assert rep["objects"]["/var/task/pkg/u_rpath.so"]["needed"][0] == {"name": "libv.so", "how": "rpath",
                                                                       "path": "/var/task/lib/libv.so"}
    assert {n["how"] for n in rep["objects"]["/var/task/pkg/u_runpath.so"]["needed"] if n["name"] == "liba.so.1"} == {"runpath"}
    # the soname symlink resolves to the one object behind it
    assert "/var/task/lib/liba.so.1.0" in rep["objects"] and rep["stats"]["rounds"] == 2


def test_rpath_loader_chain_and_runpath_not_inherited(tmp_path, emu, libs):
    entries = {"pkg/chain_rpath.so": libs["chain_rpath"], "pkg/chain_runpath.so": libs["chain_runpath"],
               "lib/libmid.so": libs["libmid"], "deep/libdeep.so": libs["libdeep"]}
    z = make_zip(str(tmp_path / "c.zip"), entries)
    rep = oracle_compare(tmp_path, z, emu, "/var/task", ["/nonexistent"])
    probs = {(p["object"], p["kind"]) for p in rep["problems"]}
    # chain_rpath: libmid finds libdeep through its loader's RPATH; chain_runpath's RUNPATH is not inherited
    assert ("/var/task/lib/libmid.so", "missing") in probs
    assert model_resolutions(rep, "/var/task/pkg/chain_rpath.so")["libdeep.so"] == "/var/task/deep/libdeep.so"
    assert model_resolutions(rep, "/var/task/pkg/chain_runpath.so")["libdeep.so"] is None


@pytest.mark.parametrize("mount,libdir", [("/var/task", "/var/task/lib"), ("/opt", "/opt/lib")])
def test_ld_library_path_lib_dirs_and_mounts(tmp_path, emu, libs, mount, libdir):
    z = make_zip(str(tmp_path / "l.zip"), {"python/pkg/u_plain.so": libs["u_plain"], "lib/liba.so.1": libs["liba"],
                                           "lib/libv.so": libs["libv"]})
    rep = oracle_compare(tmp_path, z, emu, mount, [libdir])
    assert rep["problems"] == [] and rep["mount"] == mount
    root = mount + "/python/pkg/u_plain.so"
    assert {n["how"] for n in rep["objects"][root]["needed"] if n["name"] in ("libv.so", "liba.so.1")} == {"ld_library_path"}
    # the Lambda default path names both lib directories
    rep = check(z, emu, mount=mount)
    assert rep["problems"] == [], rep["problems"]


def test_missing_arch_and_soname_match(tmp_path, emu, libs):
    z = make_zip(str(tmp_path / "m.zip"), {"pkg/u_rpath.so": libs["u_rpath"], "lib/libv.so": libs["libv"]})
    rep = oracle_compare(tmp_path, z, emu, "/var/task", ["/nonexistent"])
    assert [(p["object"], p["kind"]) for p in rep["problems"]] == [("/var/task/pkg/u_rpath.so", "missing")]
    assert "liba.so.1" in rep["problems"][0]["detail"]
    # liba found by its file name liba.so.1 whose SONAME is also liba.so.1, needed twice: one object
    z = make_zip(str(tmp_path / "arm.zip"), {"pkg/u_rpath.so": libs["u_rpath"], "lib/libv.so": libs["libv"],
                                             "lib/liba.so.1": libs["liba_arm"]})
    rep = check(z, emu)
    assert [(p["object"], p["kind"]) for p in rep["problems"]] == [("/var/task/lib/liba.so.1", "arch")]
    rep = check(z, emu, arch="arm64")
    assert {p["object"] for p in rep["problems"] if p["kind"] == "arch"} == {"/var/task/pkg/u_rpath.so",
                                                                           "/var/task/lib/libv.so"}


def test_soname_matches_an_object_already_loaded(tmp_path, emu, libs):
    """a need whose name is the SONAME of an object the root's load already holds is that object: libv's SONAME made
    liba.so.1, u_rpath's second need (liba.so.1) is then libv, not the file lib/liba.so.1"""
    z = make_zip(str(tmp_path / "s.zip"), {"pkg/u_rpath.so": libs["u_rpath"], "lib/libv.so": libs["libv"],
                                           "lib/liba.so.1": libs["liba"]})

    def rename(o):
        status, machine, recs = o
        return status, machine, [(k, f, r, "liba.so.1" if k == N.ELF_REC_SONAME and name == "libv.so" else name)
                                 for k, f, r, name in recs]
    rep = check(z, emu, edit=rename)
    got = [(r["name"], r["how"], r["path"]) for r in rep["resolved"]["/var/task/pkg/u_rpath.so"]
           if r["object"] == "/var/task/pkg/u_rpath.so"]
    assert got[:2] == [("libv.so", "rpath", "/var/task/lib/libv.so"), ("liba.so.1", "loaded", "/var/task/lib/libv.so")]
    assert "/var/task/lib/liba.so.1" not in rep["closures"]["/var/task/pkg/u_rpath.so"]


def _src(d, name, text):
    p = os.path.join(d, name)
    with open(p, "w") as f:
        f.write(text)
    return p


def test_verdef_miss_weak_and_ceilings(tmp_path, emu, libs):
    z = make_zip(str(tmp_path / "v.zip"), {"pkg/u_rpath.so": libs["u_rpath"], "lib/liba.so.1": libs["liba"],
                                           "lib/libv.so": libs["libv1only"]})
    rep = check(z, emu)
    assert [(p["kind"], p["detail"]) for p in rep["problems"]] == [("version", "V2 not defined by libv.so")]

    def weaken(o):
        status, machine, recs = o
        return status, machine, [(k, f | 2 if k == N.ELF_REC_VERNEED_VERSION and name == "V2" else f, r, name)
                                 for k, f, r, name in recs]
    rep = check(z, emu, edit=weaken)
    assert rep["problems"] == [] and [n["detail"] for n in rep["notes"]] == ["V2 not defined by libv.so"]
    # the highest glibc version needed, and a ceiling under it
    d = str(tmp_path)
    libc_user = cc(os.path.join(d, "libc_user.so"), _src(d, "c.c", "#include <stdio.h>\nint p(void) { return puts(\"x\"); }\n"))
    z = make_zip(str(tmp_path / "g.zip"), {"pkg/u_rpath.so": libs["u_rpath"], "lib/liba.so.1": libs["liba"],
                                           "lib/libv.so": libs["libv"], "pkg/libc_user.so": libc_user})
    rep = check(z, emu)
    assert rep["problems"] == [] and "GLIBC" in rep["max_versions"]
    top = rep["max_versions"]["GLIBC"]
    assert set(rep["provided_used"]) >= {"libc.so.6"}
    rep = check(z, emu, max_versions={"GLIBC": "2.0"})
    assert rep["problems"] and all(p["kind"] == "version" and "GLIBC" in p["detail"] for p in rep["problems"])
    assert check(z, emu, max_versions={"GLIBC": top})["problems"] == []
    with pytest.raises(ValueError):
        check(z, emu, max_versions={"GLIBC": "two"})


@pytest.fixture(scope="module")
def numpy_scipy_layer(tmp_path_factory):
    """the shared objects of numpy and scipy and their .libs, zipped as a layer (prefix python/)"""
    sp = F.site_packages()
    path = str(tmp_path_factory.mktemp("np_layer") / "layer.zip")
    with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as zf:
        for p in D.site_objects():
            zf.write(p, "python/" + os.path.relpath(p, sp))
    return path


def test_numpy_scipy_layer_against_the_loader(tmp_path, emu, numpy_scipy_layer):
    rep = oracle_compare(tmp_path, numpy_scipy_layer, emu, "/opt", ["/opt/lib"])
    assert rep["problems"] == []
    assert rep["stats"]["rounds"] == 3
    umath = [p for p in rep["closures"] if "_multiarray_umath" in p][0]
    gfortran = [p for p in rep["closures"][umath] if "libgfortran" in p]
    assert gfortran and gfortran[0].startswith("/opt/python/numpy.libs/")
    rep = check(numpy_scipy_layer, emu, mount="/opt")
    assert rep["max_versions"]["GLIBC"] == "2.27" and rep["problems"] == []


def test_command_exit_codes(tmp_path, emu, libs, capsys):
    ok = make_zip(str(tmp_path / "ok.zip"), {"pkg/u_rpath.so": libs["u_rpath"], "lib/liba.so.1": libs["liba"],
                                             "lib/libv.so": libs["libv"]})
    bad = make_zip(str(tmp_path / "bad.zip"), {"pkg/u_rpath.so": libs["u_rpath"]})
    run = lambda zip_path, **kw: check(zip_path, emu, **kw)  # noqa: E731
    assert deps.main([ok], check=run) == 0
    assert deps.main([bad], check=run) == 1
    out = capsys.readouterr().out
    assert "problem: /var/task/pkg/u_rpath.so: missing" in out
    assert deps.main([ok, "--json"], check=run) == 0
    capsys.readouterr()
    not_zip = str(tmp_path / "x.zip")
    with open(not_zip, "wb") as f:
        f.write(b"not a zip")
    assert deps.main([not_zip], check=run) == 2
    assert deps.main([ok, "--max-version", "GLIBC"], check=run) == 2
    assert deps.main([str(tmp_path / "absent.zip")], check=run) == 2
    with pytest.raises(SystemExit) as e:
        deps.main([ok, "--arch", "mips"], check=run)
    assert e.value.code == 2


def test_bundle_check_deps_hook(tmp_path, monkeypatch, capsys):
    from lambdipy_b200 import patch, zipfile_gpu
    monkeypatch.delenv("LAMBDIPY_BUNDLE_CHECK_DEPS", raising=False)
    assert patch.bundle_check_deps() is False
    monkeypatch.setenv("LAMBDIPY_BUNDLE_CHECK_DEPS", "1")
    assert patch.bundle_check_deps() is True
    for bad in ("0", "yes", ""):
        monkeypatch.setenv("LAMBDIPY_BUNDLE_CHECK_DEPS", bad)
        with pytest.raises(ValueError):
            patch.bundle_check_deps()
    build = tmp_path / "build"
    build.mkdir()
    (build / "a.txt").write_text("x")
    zip_path = str(tmp_path / "bundle.zip")
    monkeypatch.setattr(zipfile_gpu, "zip_tree", lambda src, dst, **kw: make_zip(dst, {"a.txt": str(build / "a.txt")}))
    reports = {"ok": {"problems": [], "stats": {"objects": 7}},
               "bad": {"problems": [{"object": "/var/task/x.so", "kind": "missing", "detail": "liby.so"}],
                       "stats": {"objects": 1, "roots": 1, "rounds": 1}, "mount": "/var/task", "arch": "x86_64",
                       "max_versions": {}, "provided_used": {}, "notes": []}}
    for key in ("ok", "bad"):
        monkeypatch.setattr(deps, "check_zip", lambda p, **kw: reports[key])
        wrapped = patch.zip_after_copy(lambda paths, d: None, zip_path, check_deps=True)
        if key == "ok":
            wrapped([], str(build))
            assert "; 7 shared objects checked" in capsys.readouterr().out
        else:
            with pytest.raises(RuntimeError, match="liby.so"):
                wrapped([], str(build))
