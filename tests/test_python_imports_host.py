"""CPU checks of check_with(python=...) behind zlib, the dynamic-section parse emulator and the symbol emulator, with
CPython's own finder as the oracle: importlib.machinery.PathFinder (its _get_spec) walked level by level over the extracted zip's
sys.path (Lambda's entries, mapped under a temporary root) with a FileFinder.path_hook built from the target's
loaders -- ExtensionFileLoader with [".cpython-3N-<triplet>.so", ".abi3.so", ".so"], then source, then bytecode --
and no package executed.  For 3.12 on x86_64 the hook is this interpreter's own (_get_supported_file_loaders).  The
PyInit_* lookups are compared with ctypes.CDLL(path, RTLD_NOW | RTLD_LOCAL) and hasattr.

Fixtures: a good module; a renamed one; a cpython-311 file alone and beside a .py; an aarch64 triplet and a -darwin
build; .abi3.so shadowed by .cpython-312; a package directory beating a .so and a namespace directory losing to one;
one top-level name in both layer path entries; pkg/__init__.cpython-312; a non-ASCII name (PyInitU_); a bare .so
module and a bare .so library; both mounts; a split decoder.  Real packages: numpy + scipy as a layer, an installed
abi3 package; python=None, refused values and the commands' exit codes."""
import ctypes
import importlib.machinery as M
import os
import sys
import zipfile

import pytest

import deps_lib as D
import elf_fixtures as F
import find_lib as FL
from lambdipy_b200 import deps
from lambdipy_b200 import layer as L
from test_deps_host import EmuParser, TableZlibDecoder, extract
from test_deps_host import check as plain_check
from test_python_imports_emulated import MOD, _cc
from test_strip_zip_host import FakeMemory

T312 = ".cpython-312-x86_64-linux-gnu.so"


def check(zip_path, emu, **kw):
    mem = FakeMemory()
    return deps.check_with(zip_path, TableZlibDecoder(mem), EmuParser(mem, emu), resolver=FL.EmuResolver(mem), **kw)


@pytest.fixture(scope="module")
def emu():
    return D.Emu()


@pytest.fixture(scope="module")
def mods(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("py_mods"))
    m = {}
    for name in ("good", "old311", "both311", "armmod", "mac", "shadow", "dirwins", "nsloses", "dup", "ipkg", "bare"):
        m[name] = _cc(d, name + ".so", MOD % name)
    m["renamed"] = _cc(d, "renamed.so", MOD % "original")
    m["cafe"] = _cc(d, "cafe.so", MOD.replace("PyInit_%s", "PyInitU_%s") % "caf_dma")
    m["libhelper"] = _cc(d, "libhelper.so", "int helper(void) { return 1; }\n")
    return m


def write_zip(path, members):
    """members {name: file path or bytes}"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for name, src in members.items():
            if isinstance(src, bytes):
                zf.writestr(name, src)
            else:
                zf.write(src, name)
    return path


def function_zip(tmp_path, m):
    return write_zip(str(tmp_path / "fn.zip"), {
        "good" + T312: m["good"], "renamed" + T312: m["renamed"],
        "old311.cpython-311-x86_64-linux-gnu.so": m["old311"],
        "both311.cpython-311-x86_64-linux-gnu.so": m["both311"], "both311.py": b"x = 1\n",
        "armmod.cpython-312-aarch64-linux-gnu.so": m["armmod"], "mac.cpython-312-darwin.so": m["mac"],
        "pkg3/__init__.py": b"", "pkg3/shadow.abi3.so": m["shadow"], "pkg3/shadow" + T312: m["shadow"],
        "dirwins/__init__.py": b"", "dirwins" + T312: m["dirwins"],
        "nsloses/data.txt": b"data", "nsloses" + T312: m["nsloses"],
        "ipkg/__init__" + T312: m["ipkg"], "café" + T312: m["cafe"],
        "bare.so": m["bare"], "lib/libhelper.so": m["libhelper"], "numpy.libs/libx.so": m["libhelper"]})


def layer_zip(tmp_path, m):
    return write_zip(str(tmp_path / "layer.zip"), {
        "python/lib/python3.12/site-packages/dup" + T312: m["dup"], "python/dup" + T312: m["dup"],
        "python/good" + T312: m["good"]})


def oracle(root, version, arch, mount):
    """{dotted name: mounted origin or None}: a function that finds names as CPython does over root + sys.path"""
    minor, trip = version.split(".")[1], deps.TRIPLETS[arch]
    ext = [".cpython-3%s-%s.so" % (minor, trip), ".abi3.so", ".so"]
    if (version, arch) == ("3.12", "x86_64") and sys.version_info[:2] == (3, 12):
        assert M.EXTENSION_SUFFIXES == ext
        import importlib._bootstrap_external as BE
        loaders = BE._get_supported_file_loaders()
    else:
        loaders = [(M.ExtensionFileLoader, ext), (M.SourceFileLoader, M.SOURCE_SUFFIXES),
                   (M.SourcelessFileLoader, M.BYTECODE_SUFFIXES)]
    hook = M.FileFinder.path_hook(*loaders)
    path = [root + p.format(version=version) for p in deps.LAMBDA_PYTHON_PATH
            if p.format(version=version).startswith(mount.rstrip("/") + "/") or p == mount]

    def find(dotted):
        saved = sys.path_hooks, sys.path_importer_cache
        sys.path_hooks, sys.path_importer_cache = [hook], {}
        try:
            parts, search, spec = dotted.split("."), path, None
            for i in range(len(parts)):
                if i:
                    if spec is None or spec.submodule_search_locations is None:
                        return None
                    search = list(spec.submodule_search_locations)
                # find_spec less its last step, which wraps a namespace's portions in a _NamespacePath that looks
                # its parent up in sys.modules: nothing here is imported
                spec = M.PathFinder._get_spec(".".join(parts[:i + 1]), search)
                if spec is not None and spec.loader is None and not spec.submodule_search_locations:
                    spec = None
            if spec is None:
                return None
            return spec.origin[len(root):] if spec.origin and spec.has_location else "namespace"
        finally:
            sys.path_hooks, sys.path_importer_cache = saved
    return find


def compare_with_cpython(tmp_path, zip_path, rep, version, mount, arch="x86_64"):
    root = str(tmp_path / ("tree_" + version.replace(".", "_")))
    if not os.path.isdir(root):
        extract(zip_path, root + mount)
    find = oracle(root, version, arch, mount)
    for p, rec in rep["python"]["modules"].items():
        if rec["module"] is None:
            continue
        got = find(rec["module"])
        if rec["class"] in ("module", "library"):  # a library here is a bare .so the finder loads without PyInit_*
            assert got == p, (p, rec, got)
        elif rec["class"] == "shadowed":
            assert got != p, (p, rec, got)
        else:
            problem = any(x["object"] == p and x["kind"] == "python" for x in rep["problems"])
            assert problem == (got is None), (p, rec, got)
        if rec["class"] == "module" and rec["status"] in ("ok", "not exported"):
            lib = ctypes.CDLL(root + p, os.RTLD_NOW | os.RTLD_LOCAL)
            assert hasattr(lib, rec["export"]) == (rec["status"] == "ok"), (p, rec)
    return root


def classes(rep):
    return {p: (r["class"], r["status"]) for p, r in rep["python"]["modules"].items()}


def test_fixtures_against_cpython(tmp_path, emu, mods):
    z = function_zip(tmp_path, mods)
    rep = check(z, emu, python="3.12")
    compare_with_cpython(tmp_path, z, rep, "3.12", "/var/task")
    c, t = classes(rep), "/var/task/"
    assert c[t + "good" + T312] == ("module", "ok") and c[t + "renamed" + T312] == ("module", "not exported")
    assert rep["python"]["modules"][t + "good" + T312]["defined_by"] == t + "good" + T312
    assert c[t + "old311.cpython-311-x86_64-linux-gnu.so"][0] == "other python"
    assert c[t + "armmod.cpython-312-aarch64-linux-gnu.so"][0] == "other python"
    assert c[t + "pkg3/shadow.abi3.so"][0] == "shadowed" and c[t + "pkg3/shadow" + T312] == ("module", "ok")
    assert c[t + "dirwins" + T312][0] == "shadowed" and c[t + "nsloses" + T312] == ("module", "ok")
    assert c[t + "ipkg/__init__" + T312] == ("module", "ok")
    assert rep["python"]["modules"][t + "ipkg/__init__" + T312]["module"] == "ipkg"
    cafe = rep["python"]["modules"][t + "café" + T312]
    assert cafe["export"] == "PyInitU_caf_dma" and cafe["status"] == "ok"
    assert c[t + "bare.so"] == ("module", "ok")
    assert c[t + "lib/libhelper.so"] == ("library", None) and c[t + "numpy.libs/libx.so"] == ("library", None)
    probs = {(p["object"][len(t):], p["detail"]) for p in rep["problems"] if p["kind"] == "python"}
    assert probs == {
        ("renamed" + T312, 'PyInit_renamed not exported: the import fails with "dynamic module does not define module '
                           'export function"'),
        ("old311.cpython-311-x86_64-linux-gnu.so",
         "old311: built only for cpython-311-x86_64-linux-gnu; Python 3.12 finds no module old311"),
        ("armmod.cpython-312-aarch64-linux-gnu.so",
         "armmod: built only for cpython-312-aarch64-linux-gnu; Python 3.12 finds no module armmod"),
        ("mac.cpython-312-darwin.so", "mac: built only for cpython-312-darwin; Python 3.12 finds no module mac")}
    notes = {p["object"][len(t):] for p in rep["notes"] if p["kind"] == "python"}
    assert notes == {"both311.cpython-311-x86_64-linux-gnu.so", "pkg3/shadow.abi3.so", "dirwins" + T312}
    st = rep["stats"]
    assert st["modules"] == 7 and st["python_skipped"] == 0 and st["find_queries"] == 8  # + lib/libhelper.so
    assert rep["python"]["path"] == ["/var/task", "/opt/python/lib/python3.12/site-packages", "/opt/python"]
    # another target: the same zip for 3.11 on arm64, against CPython's finder with those suffixes
    rep = check(z, emu, python="3.11", arch="arm64")
    compare_with_cpython(tmp_path, z, rep, "3.11", "/var/task", "arm64")
    assert classes(rep)[t + "good" + T312][0] == "other python"
    assert classes(rep)[t + "armmod.cpython-312-aarch64-linux-gnu.so"][0] == "other python"
    # a split decoder gives the same report
    mem = FakeMemory()
    split = deps.check_with(z, TableZlibDecoder(mem), EmuParser(mem, emu), resolver=FL.EmuResolver(mem), python="3.12",
                            batch_bytes=1)
    whole = check(z, emu, python="3.12")
    for r in (split, whole):
        r.pop("stats")
    assert split == whole


def test_layer_path_entries_and_both_mounts(tmp_path, emu, mods):
    z = layer_zip(tmp_path, mods)
    rep = check(z, emu, mount="/opt", python="3.12")
    compare_with_cpython(tmp_path, z, rep, "3.12", "/opt")
    c = classes(rep)
    assert c["/opt/python/lib/python3.12/site-packages/dup" + T312] == ("module", "ok")
    assert c["/opt/python/dup" + T312][0] == "shadowed" and c["/opt/python/good" + T312] == ("module", "ok")
    assert rep["problems"] == []
    # for 3.11 the site-packages entry is another directory: the 3.12 one is no module's, /opt/python's is the 3.12 build
    rep = check(z, emu, mount="/opt", python="3.11")
    assert classes(rep)["/opt/python/lib/python3.12/site-packages/dup" + T312] == ("library", None)
    assert classes(rep)["/opt/python/dup" + T312][0] == "other python"
    # the same zip as a function bundle: its python/ directory is a namespace package on /var/task
    rep = check(z, emu, python="3.12")
    compare_with_cpython(tmp_path / "fn", z, rep, "3.12", "/var/task")
    assert rep["python"]["modules"]["/var/task/python/dup" + T312]["module"] == "python.dup"
    assert classes(rep)["/var/task/python/lib/python3.12/site-packages/dup" + T312] == ("library", None)


def test_python_none_refused_and_symbols_together(tmp_path, emu, mods):
    z = function_zip(tmp_path, mods)
    base = plain_check(z, emu)
    assert "python" not in base and set(base["stats"]) == {"members", "roots", "objects", "rounds", "bytes_up",
                                                            "bytes_down", "inflate_ms", "parse_ms"}
    withp = check(z, emu, python="3.12")
    for k in ("objects", "closures", "resolved", "max_versions", "provided_used"):
        assert withp[k] == base[k]
    assert [p for p in withp["problems"] if p["kind"] != "python"] == base["problems"]
    both = check(z, emu, python="3.12", symbols=True)
    assert both["python"] == withp["python"] and "symbols" in both
    for bad in ("3.7", "3.15", "3.13t", 3.12, "312", ""):
        with pytest.raises(ValueError):
            check(z, emu, python=bad)
        with pytest.raises(ValueError):
            deps.check_options({"python": bad})
    with pytest.raises(ValueError):
        deps.check_with(z, None, None, python="3.12")  # a resolver is needed


@pytest.fixture(scope="module")
def site_layer(tmp_path_factory):
    sp = F.site_packages()
    layer = str(tmp_path_factory.mktemp("py_site") / "layer.zip")
    with zipfile.ZipFile(layer, "w", zipfile.ZIP_STORED) as zf:
        for p in D.site_objects():
            zf.write(p, "python/" + os.path.relpath(p, sp))
    return layer


def test_numpy_scipy_layer_and_commands(tmp_path, emu, site_layer, capsys):
    rep = check(site_layer, emu, mount="/opt", python="3.12")
    assert [p for p in rep["problems"] if p["kind"] == "python"] == []
    mods = rep["python"]["modules"]
    tagged = [p for p in mods if ".cpython-" in p.rsplit("/", 1)[1]]
    assert len(tagged) > 50 and all(mods[p]["class"] == "module" and mods[p]["status"] == "ok" for p in tagged)
    compare_with_cpython(tmp_path, site_layer, rep, "3.12", "/opt")
    rep = check(site_layer, emu, mount="/opt", python="3.11")
    assert {p["object"] for p in rep["problems"] if p["kind"] == "python"} == set(tagged)
    run = lambda zip_path, **kw: check(zip_path, emu, **kw) if kw.get("python") else plain_check(zip_path, emu, **kw)  # noqa: E731
    assert deps.main([site_layer, "--mount", "/opt", "--python", "3.11"], check=run) == 1
    out = capsys.readouterr().out
    assert "python 3.11:" in out and "_multiarray_umath: built only for cpython-312-x86_64-linux-gnu" in out
    assert deps.main([site_layer, "--mount", "/opt", "--python", "3.12"], check=run) == 0
    assert deps.main([site_layer, "--mount", "/opt", "--python", "3.7"], check=run) == 2


def test_abi3_package_imports_on_311_and_312(tmp_path, emu):
    sp = F.site_packages()
    pkg = next((d for d in ("psutil", "nacl", "safetensors") if any(f.endswith(".abi3.so") for f in
                                                                    os.listdir(os.path.join(sp, d)))
                if os.path.isdir(os.path.join(sp, d))), None) if os.path.isdir(sp) else None
    if pkg is None:
        pytest.skip("no installed abi3 package")
    z = str(tmp_path / "abi3.zip")
    with zipfile.ZipFile(z, "w", zipfile.ZIP_DEFLATED) as zf:
        for d, _, fs in os.walk(os.path.join(sp, pkg)):
            for f in fs:
                if "__pycache__" not in d:
                    zf.write(os.path.join(d, f), os.path.relpath(os.path.join(d, f), sp))
    for v in ("3.11", "3.12"):
        rep = check(z, emu, python=v)
        mods = rep["python"]["modules"]
        abi3 = [p for p in mods if p.endswith(".abi3.so")]
        assert abi3 and all(mods[p]["status"] == "ok" for p in abi3), (v, mods)
        assert [p for p in rep["problems"] if p["kind"] == "python"] == []


def test_layer_command_takes_python(monkeypatch):
    seen = {}
    report = {"arch": "x86_64", "mount": "/opt", "max_versions": {}, "provided_used": {}, "problems": [], "notes": [],
              "python": {"version": "3.12"},
              "stats": {"objects": 3, "roots": 2, "rounds": 2, "modules": 2, "python_skipped": 0, "find_queries": 2}}
    st = {"zip_bytes": 4e6, "src_bytes": 5e6, "entries": 12, "gpu": 3, "fallback": 0, "in_bytes": 5e6,
          "out_bytes": 1e6, "copied": {"members": 7}, "removed": {"entries": 2}, "check": report}

    def fake(dst, tarballs, wheels, prefix="", keep_tests=(), compresslevel=None, seek_table=False, check=None):
        deps.check_options(check)
        seen.update(check=check)
        if check["python"] == "3.11":
            raise deps.CheckFailed(dict(report, problems=[{"object": "/opt/python/m" + T312, "kind": "python",
                                                          "detail": "m: built only for cpython-312-x86_64-linux-gnu"}]))
        return st
    monkeypatch.setattr(L, "zip_build", fake)
    base = ["l.zip", "--wheel", "a.whl", "--prefix", "python/", "--check", "--mount", "/opt"]
    assert L.main(base + ["--python", "3.12"]) == 0 and seen["check"]["python"] == "3.12"
    assert L.main(base + ["--python", "3.11"]) == 1
    assert L.main(base + ["--python", "3.6"]) == 2
    with pytest.raises(SystemExit) as e:
        L.main(["l.zip", "--wheel", "a.whl", "--python", "3.12"])
    assert e.value.code == 2
    assert "python" in deps.CHECK_KEYS
    with pytest.raises(ValueError):
        L._check_engines({"python": "3.12"}, object(), None)  # the import check needs a resolver
