"""CPU checks of check_with(symbols=True) behind zlib, the emulator of the dynamic-section parse and the emulator of the
symbol index and lookup (tests/emu/syms_emu.cpp over elf_syms.cuh), with the real glibc loader as the oracle:

* oracle 1: `LD_TRACE_LOADED_OBJECTS=1 LD_WARN=yes LD_BIND_NOW=yes ld.so --library-path P ROOT` on the extracted zip
  prints every strong "undefined symbol" of ROOT's load; with interpreter=(), the Py* rule off and runtime_libs the
  host's library directory, the "symbol" problems equal those lines, root by root;
* oracle 2: `ctypes.CDLL(root, RTLD_NOW)` in a fresh python fails exactly for the roots the check with
  interpreter=[sys.executable] reports a problem for, naming one of the symbols reported.

Fixtures, linked by gcc here: a strong and a weak missing reference, a reference left to a sibling module outside the
scope, the three hash styles, packed relative relocations, a version script with f@@V2 and a hidden f@V1 and users
of V1, an unversioned user of a hidden-only version, TLS / IFUNC / GNU_UNIQUE / protected definitions, a missing
DT_NEEDED, and an unversioned name only libz.so.1 defines."""
import json
import os
import re
import subprocess
import sys
import zipfile

import pytest

import deps_lib as D
import elf_fixtures as F
import syms_lib as S
from lambdipy_b200 import deps
from test_deps_host import EmuParser, TableZlibDecoder, extract, make_zip
from test_deps_host import check as plain_check
from test_strip_zip_host import FakeMemory

LD_SO = "/lib64/ld-linux-x86-64.so.2"
HOST_LIBS = "/lib/x86_64-linux-gnu"


def check(zip_path, emu, **kw):
    mem = FakeMemory()
    return deps.check_with(zip_path, TableZlibDecoder(mem), EmuParser(mem, emu), symbols=True,
                           resolver=S.EmuResolver(mem), **kw)


@pytest.fixture(scope="module")
def emu():
    return D.Emu()


def _cc(d, out, code, *args):
    src = os.path.join(d, out + ".c")
    with open(src, "w") as f:
        f.write(code)
    p = os.path.join(d, out)
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-o", p, src] + list(args), check=True, capture_output=True)
    return p


@pytest.fixture(scope="module")
def fx(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("syms_fx"))
    L = {}
    full = "int a_fn(void) { return 1; }\nint b_fn(void) { return 2; }\n"
    for style in ("gnu", "sysv", "both"):
        L["def_" + style] = _cc(d, "libdef_%s.so" % style, full, "-Wl,-soname,libdef.so", "-Wl,--hash-style=" + style)
    L["def_noB"] = _cc(d, "libdef_nob.so", "int a_fn(void) { return 1; }\n", "-Wl,-soname,libdef.so")
    user = ("int a_fn(void); int b_fn(void); __attribute__((weak)) int w_fn(void);\n"
            "int use(void) { return a_fn() + b_fn() + (w_fn ? w_fn() : 0); }\n")
    L["user"] = _cc(d, "user.so", user, "-L" + d, "-l:libdef_gnu.so")
    L["user_relr"] = _cc(d, "user_relr.so", user + "static int *ptrs[] = {0, 0};\nint **pp(void) { return ptrs; }\n",
                         "-L" + d, "-l:libdef_gnu.so", "-Wl,-z,pack-relative-relocs")
    L["sib_a"] = _cc(d, "sib_a.so", "int sib_fn(void) { return 7; }\n")
    L["sib_b"] = _cc(d, "sib_b.so", "int sib_fn(void);\nint sb(void) { return sib_fn(); }\n")
    # versions: f@@V2 and a hidden f@V1; an old library with V1 only; users of each
    v2 = ("int f_v1(void) { return 1; }\nint f_v2(void) { return 2; }\n"
          "__asm__(\".symver f_v1,f@V1\");\n__asm__(\".symver f_v2,f@@V2\");\n")
    L["ver_new"] = _cc(d, "libver.so", v2, "-Wl,--version-script=" + _w(d, "v.map", "V1 { local: f_v*; };\nV2 { } V1;\n"),
                       "-Wl,-soname,libver.so")
    os.makedirs(os.path.join(d, "old"))
    L["ver_old"] = _cc(os.path.join(d, "old"), "libver.so", "int f(void) { return 1; }\n",
                       "-Wl,--version-script=" + _w(d, "v1.map", "V1 { global: f; local: *; };\n"), "-Wl,-soname,libver.so")
    L["ver_user"] = _cc(d, "ver_user.so", "int f(void);\nint vu(void) { return f(); }\n", "-L" + os.path.join(d, "old"), "-lver")
    L["ver_nov1"] = _cc(d, "libver_nov1.so", "int f(void) { return 2; }\n",
                        "-Wl,--version-script=" + _w(d, "v2.map", "V2 { global: f; local: *; };\n"), "-Wl,-soname,libver.so")
    # an unversioned user of a library whose only definition of g is hidden-versioned (g@V1, not the default)
    # (V0 takes versym index 2, which an unversioned reference takes directly; g is at V1, index 3)
    hmap = _w(d, "h.map", "V0 { global: h0; local: g_impl; };\nV1 { } V0;\n")
    L["hid_lib"] = _cc(d, "libhid.so", "int h0 = 1;\nint g_impl(void) { return 3; }\n__asm__(\".symver g_impl,g@V1\");\n",
                       "-Wl,--version-script=" + hmap, "-Wl,-soname,libhid.so")
    # the same with g@@V1: the default, not hidden, and the object's single candidate -- taken
    L["hid_default"] = _cc(d, "libhid_default.so", "int h0 = 1;\nint g_impl(void) { return 3; }\n"
                                                   "__asm__(\".symver g_impl,g@@V1\");\n",
                           "-Wl,--version-script=" + hmap, "-Wl,-soname,libhid.so")
    L["hid_stub"] = _cc(d, "libhid_stub.so", "int g(void) { return 0; }\n", "-Wl,-soname,libhid.so")
    L["hid_user"] = _cc(d, "hid_user.so", "int g(void);\nint hu(void) { return g(); }\n", "-L" + d, "-l:libhid_stub.so")
    # TLS, IFUNC, GNU_UNIQUE (a C++ inline static local) and protected definitions, and their user
    kinds = ("__thread int tls_v = 1;\nstatic int impl(void) { return 4; }\nstatic void *res(void) { return (void *)impl; }\n"
             "int ifn(void) __attribute__((ifunc(\"res\")));\n__attribute__((visibility(\"protected\"))) int prot_fn(void) { return 5; }\n")
    L["kinds"] = _cc(d, "libkinds.so", kinds, "-Wl,-soname,libkinds.so")
    L["uniq"] = _cc(d, "libuniq.so", "", "-x", "c++", "-")  # placeholder replaced below
    os.remove(L["uniq"])
    src = _w(d, "uniq.cc", "template <class T> struct S { static int &v() { static int x = 6; return x; } };\n"
                            "extern \"C\" int uq(void) { return S<int>::v(); }\n")
    L["uniq"] = os.path.join(d, "libuniq.so")
    subprocess.run(["g++", "-shared", "-fPIC", "-O1", "-o", L["uniq"], src, "-Wl,-soname,libuniq.so"], check=True)
    L["kinds_user"] = _cc(d, "kinds_user.so", "extern __thread int tls_v; int ifn(void); int prot_fn(void); int uq(void);\n"
                                              "int ku(void) { return tls_v + ifn() + prot_fn() + uq(); }\n",
                          "-L" + d, "-lkinds", "-luniq")
    L["needs_gone"] = _cc(d, "needs_gone.so", "int gone(void);\nint ng(void) { return gone(); }\n", "-L" + d,
                          "-Wl,--no-as-needed", "-l:libgone.so") if _cc(d, "libgone.so", "int gone(void) { return 0; }\n",
                                                                         "-Wl,-soname,libgone.so") else None
    # an unversioned reference that only libz.so.1 defines (crc32 at zlib's base version)
    L["z_stub"] = _cc(d, "libz_stub.so", "unsigned long crc32(unsigned long c, const unsigned char *b, unsigned n) { return 0; }\n",
                      "-Wl,-soname,libz.so.1")
    L["z_user"] = _cc(d, "z_user.so", "unsigned long crc32(unsigned long, const unsigned char *, unsigned);\n"
                                      "unsigned long zu(void) { return crc32(0, 0, 0); }\n", "-L" + d, "-l:libz_stub.so")
    return L


def _w(d, name, text):
    p = os.path.join(d, name)
    with open(p, "w") as f:
        f.write(text)
    return p


def ld_trace(root_file, library_path):
    """{(object path, symbol name)} of the strong undefined symbols the loader's trace prints for ROOT"""
    env = dict(os.environ, LD_TRACE_LOADED_OBJECTS="1", LD_WARN="yes", LD_BIND_NOW="yes")
    r = subprocess.run([LD_SO, "--library-path", library_path, root_file], capture_output=True, text=True, env=env)
    out = set()
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"undefined symbol: ([^\s,]+)(?:, version (\S+))?\s+\((.*)\)", line)
        if m:
            out.add((os.path.normpath(m.group(3)), m.group(1) + ("@" + m.group(2) if m.group(2) else "")))
    return out


def symbol_problems(report):
    """{(object, NAME[@VERSION], root)} of the "symbol" problems"""
    out = set()
    for p in report["problems"]:
        if p["kind"] == "symbol" and "no definition" in p["detail"]:
            m = re.match(r"(\S+): no definition in the load scope of (\S+)$", p["detail"])
            out.add((p["object"], m.group(1), m.group(2)))
    return out


def oracle_trace(tmp_path, zip_path, emu, mount="/var/task"):
    tree = str(tmp_path / "tree")
    extract(zip_path, tree + mount)
    rep = check(zip_path, emu, mount=mount, ld_library_path=mount + "/lib", runtime_libs=[HOST_LIBS],
                python_names=False)
    got = symbol_problems(rep)
    for root in rep["closures"]:
        if any(r["how"] == "missing" for r in rep["resolved"][root]):
            continue
        want = {(o[len(tree):], s) for o, s in ld_trace(tree + root, tree + mount + "/lib")}
        mine = {(o, s) for o, s, r in got if r == root}
        # a problem is reported once per (object, symbol), under the first root that met it
        assert mine <= want, (root, mine, want)
        assert want <= {(o, s) for o, s, _ in got}, (root, want, got)
    return rep


def test_mismatch_weak_sibling_and_hash_styles(tmp_path, emu, fx):
    z = make_zip(str(tmp_path / "a.zip"), {"pkg/user.so": fx["user"], "lib/libdef.so": fx["def_noB"],
                                           "pkg/sib_a.so": fx["sib_a"], "pkg/sib_b.so": fx["sib_b"],
                                           "pkg/user_relr.so": fx["user_relr"]})
    rep = oracle_trace(tmp_path, z, emu)
    got = {(o, s) for o, s, _ in symbol_problems(rep)}
    assert got == {("/var/task/pkg/user.so", "b_fn"), ("/var/task/pkg/user_relr.so", "b_fn"),
                   ("/var/task/pkg/sib_b.so", "sib_fn")}
    s = rep["symbols"]["/var/task/pkg/user.so"]
    assert s["references"] >= 3 and s["in_zip"] == 1  # a_fn; b_fn is missing, the weak ones count nowhere
    assert rep["stats"]["references"] > 0 and rep["stats"]["lookups"] > 0
    for style in ("gnu", "sysv", "both"):
        z = make_zip(str(tmp_path / ("h_%s.zip" % style)), {"pkg/user.so": fx["user"], "lib/libdef.so": fx["def_" + style]})
        rep = check(z, emu, ld_library_path="/var/task/lib")
        assert rep["problems"] == [] and rep["symbols"]["/var/task/pkg/user.so"]["in_zip"] == 2, style


def test_versions_hidden_and_num_versions(tmp_path, emu, fx):
    z = make_zip(str(tmp_path / "v.zip"), {"pkg/ver_user.so": fx["ver_user"], "lib/libver.so": fx["ver_new"],
                                           "pkg/hid_user.so": fx["hid_user"], "lib/libhid.so": fx["hid_lib"]})
    rep = oracle_trace(tmp_path, z, emu)
    # f@V1 is hidden in the new library but matches a V1 reference; g@V1 is hidden, so the unversioned user misses it
    assert {(o, s) for o, s, _ in symbol_problems(rep)} == {("/var/task/pkg/hid_user.so", "g")}
    assert rep["symbols"]["/var/task/pkg/ver_user.so"]["in_zip"] == 1
    z = make_zip(str(tmp_path / "v1.zip"), {"pkg/hid_user.so": fx["hid_user"], "lib/libhid.so": fx["hid_default"]})
    rep = oracle_trace(tmp_path / "1", z, emu)
    assert symbol_problems(rep) == set() and rep["symbols"]["/var/task/pkg/hid_user.so"]["in_zip"] == 1
    z = make_zip(str(tmp_path / "v2.zip"), {"pkg/ver_user.so": fx["ver_user"], "lib/libver.so": fx["ver_nov1"]})
    rep = oracle_trace(tmp_path / "2", z, emu)
    assert {(o, s) for o, s, _ in symbol_problems(rep)} == {("/var/task/pkg/ver_user.so", "f@V1")}


def test_symbol_kinds_and_missing_needed(tmp_path, emu, fx):
    z = make_zip(str(tmp_path / "k.zip"), {"pkg/kinds_user.so": fx["kinds_user"], "lib/libkinds.so": fx["kinds"],
                                           "lib/libuniq.so": fx["uniq"], "pkg/needs_gone.so": fx["needs_gone"]})
    rep = oracle_trace(tmp_path, z, emu)
    assert symbol_problems(rep) == set()
    assert rep["symbols"]["/var/task/pkg/kinds_user.so"]["in_zip"] >= 4
    assert rep["stats"]["symbols_skipped"] == 1 and "/var/task/pkg/needs_gone.so" not in rep["symbols"]


def test_libz_runtime_or_unverified(tmp_path, emu, fx):
    z = make_zip(str(tmp_path / "z.zip"), {"pkg/z_user.so": fx["z_user"]})
    rep = check(z, emu, runtime_libs=[HOST_LIBS])
    assert rep["problems"] == [] and rep["symbols"]["/var/task/pkg/z_user.so"]["runtime"] >= 1
    rep = check(z, emu)
    assert rep["problems"] == [] and rep["symbols"]["/var/task/pkg/z_user.so"]["unverified"] == 1
    assert [n["kind"] for n in rep["notes"]] == ["symbol"] and "libz.so.1" in rep["notes"][0]["detail"]
    # without libz.so.1 among the provided libraries the need is missing and the root is not symbol-checked
    rep = check(z, emu, provided=deps.DEFAULT_PROVIDED - {"libz.so.1"})
    assert any(p["kind"] == "missing" for p in rep["problems"]) and rep["stats"]["symbols_skipped"] == 1


def test_ctypes_load_fails_exactly_where_reported(tmp_path, emu, fx):
    z = make_zip(str(tmp_path / "c.zip"), {"pkg/user.so": fx["user"], "lib/libdef.so": fx["def_noB"],
                                           "pkg/sib_b.so": fx["sib_b"], "pkg/kinds_user.so": fx["kinds_user"],
                                           "lib/libkinds.so": fx["kinds"], "lib/libuniq.so": fx["uniq"],
                                           "pkg/z_user.so": fx["z_user"]})
    tree = str(tmp_path / "tree")
    extract(z, tree + "/var/task")
    rep = check(z, emu, ld_library_path="/var/task/lib", interpreter=[sys.executable], runtime_libs=[HOST_LIBS])
    reported = {}
    for p in rep["problems"]:
        if p["kind"] == "symbol":
            m = re.match(r"(\S+): no definition in the load scope of (\S+)$", p["detail"])
            reported.setdefault(m.group(2), set()).add(m.group(1).split("@")[0])
    for root in rep["closures"]:
        code = "import ctypes, os, sys\ntry:\n ctypes.CDLL(os.path.abspath(sys.argv[1]), os.RTLD_NOW)\nexcept OSError as e:\n print(e)"
        r = subprocess.run([sys.executable, "-c", code, tree + root], capture_output=True, text=True,
                           env=dict(os.environ, LD_LIBRARY_PATH=tree + "/var/task/lib"))
        m = re.search(r"undefined symbol: (\S+?)(?:,|$)", r.stdout.strip())
        assert bool(m) == (root in reported), (root, r.stdout, reported)
        if m:
            assert m.group(1) in reported[root]


def test_numpy_scipy_layer_and_command(tmp_path, emu, fx, capsys):
    sp = F.site_packages()
    layer = str(tmp_path / "layer.zip")
    with zipfile.ZipFile(layer, "w", zipfile.ZIP_STORED) as zf:
        for p in D.site_objects():
            zf.write(p, "python/" + os.path.relpath(p, sp))
    rep = check(layer, emu, mount="/opt")
    assert rep["problems"] == [], rep["problems"][:5]
    umath = [p for p in rep["symbols"] if "_multiarray_umath" in p][0]
    assert rep["symbols"][umath]["interpreter"] > 100 and rep["symbols"][umath]["trusted"] > 10
    # with the host's libraries read, the same holds and references bind to them
    rep = check(layer, emu, mount="/opt", runtime_libs=[HOST_LIBS])
    assert rep["problems"] == [], rep["problems"][:5] and rep["symbols"][umath]["runtime"] > 10
    base = plain_check(layer, emu, mount="/opt")
    assert "symbols" not in base and set(base["stats"]) == {"members", "roots", "objects", "rounds", "bytes_up",
                                                             "bytes_down", "inflate_ms", "parse_ms"}
    # the command: exit codes with and without --symbols
    bad = make_zip(str(tmp_path / "bad.zip"), {"pkg/user.so": fx["user"], "lib/libdef.so": fx["def_noB"]})
    run = lambda zip_path, **kw: check(zip_path, emu, **kw) if kw.pop("symbols", False) else \
        plain_check(zip_path, emu, **kw)  # noqa: E731
    assert deps.main([bad, "--ld-library-path", "/var/task/lib"], check=run) == 0
    assert deps.main([bad, "--ld-library-path", "/var/task/lib", "--symbols"], check=run) == 1
    out = capsys.readouterr().out
    assert "problem: /var/task/pkg/user.so: symbol: b_fn: no definition in the load scope of /var/task/pkg/user.so" in out
    assert deps.main([bad, "--ld-library-path", "/var/task/lib", "--symbols", "--runtime-lib", HOST_LIBS,
                      "--interpreter", sys.executable, "--json"], check=run) == 1
    assert json.loads(capsys.readouterr().out)["stats"]["symbols_skipped"] == 0
