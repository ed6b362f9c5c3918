"""CPU checks of lb2_syms_find's logic without a GPU: elf_syms.cuh's lookup_name under g++
(tests/emu/syms_find_emu.cpp), looking PyInit_* names up as dlsym does, against the real dlsym: `ctypes.CDLL(path, RTLD_NOW | RTLD_LOCAL)` and
`hasattr(lib, name)` on extension modules gcc builds here against Python.h.

Fixtures: a plain module; PyInit as the default version @@V1 (found) and only as a hidden @V1 (not found); a version
script with `local: *` (not found); a weak definition; an STT_OBJECT named PyInit_x (found, as dlsym finds it);
PyInit defined only in an $ORIGIN DT_NEEDED library (found through the local scope) and only in a library outside the
closure (not found); the three hash styles.  An ASan + UBSan build then looks names up in the existing mutants and
with names at the pool's edges."""
import ctypes
import os
import subprocess
import sysconfig

import pytest

import deps_lib as D
import find_lib as FL
from lambdipy_b200 import deps
from test_elf_syms_emulated import symbol_mutants

PY_INC = sysconfig.get_paths()["include"]
MOD = '#include <Python.h>\nPyMODINIT_FUNC PyInit_%s(void) { return NULL; }\n'


def _w(d, name, text):
    p = os.path.join(d, name)
    with open(p, "w") as f:
        f.write(text)
    return p


def _cc(d, out, code, *args):
    p = os.path.join(d, out)
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-I" + PY_INC, "-o", p, _w(d, out + ".c", code)] + list(args),
                   check=True, capture_output=True)
    return p


@pytest.fixture(scope="module")
def fx(tmp_path_factory):
    """{label: (module path, [paths of its local scope after it], the name looked up)}"""
    if not os.path.exists(os.path.join(PY_INC, "Python.h")):
        pytest.skip("no Python.h")
    d = str(tmp_path_factory.mktemp("pyinit_fx"))
    F = {}
    F["plain"] = (_cc(d, "plain.so", MOD % "plain"), [], "PyInit_plain")
    F["default_v1"] = (_cc(d, "dv.so", MOD % "dv", "-Wl,--version-script=" + _w(d, "dv.map", "V1 { global: PyInit_dv; local: *; };\n")),
                       [], "PyInit_dv")
    hid = ("#include <Python.h>\nint h0 = 1;\nPyObject *impl(void) { return NULL; }\n"
           "__asm__(\".symver impl,PyInit_hid@V1\");\n")
    F["hidden_v1"] = (_cc(d, "hid.so", hid, "-Wl,--version-script=" + _w(d, "h.map", "V0 { global: h0; local: impl; };\nV1 { } V0;\n")),
                      [], "PyInit_hid")
    F["local_all"] = (_cc(d, "loc.so", MOD % "loc", "-Wl,--version-script=" + _w(d, "l.map", "{ local: *; };\n")), [], "PyInit_loc")
    F["weak"] = (_cc(d, "weak.so", "#include <Python.h>\n__attribute__((weak)) PyMODINIT_FUNC PyInit_weak(void) { return NULL; }\n"),
                 [], "PyInit_weak")
    F["object"] = (_cc(d, "obj.so", "int PyInit_obj = 7;\n"), [], "PyInit_obj")
    dep = _cc(d, "libinit_dep.so", MOD % "viadep", "-Wl,-soname,libinit_dep.so")
    F["via_needed"] = (_cc(d, "viadep.so", "int other(void) { return 1; }\n", "-L" + d, "-Wl,--no-as-needed",
                           "-l:libinit_dep.so", "-Wl,-rpath,$ORIGIN"), [dep], "PyInit_viadep")
    _cc(d, "libsibling.so", MOD % "lonely")
    F["outside_closure"] = (_cc(d, "lonely.so", "int lonely(void) { return 2; }\n"), [], "PyInit_lonely")
    for style in ("gnu", "sysv", "both"):
        F["hash_" + style] = (_cc(d, "h_%s.so" % style, MOD % ("h_" + style), "-Wl,--hash-style=" + style), [],
                              "PyInit_h_" + style)
    return F


def dlsym_finds(path, name):
    lib = ctypes.CDLL(path, os.RTLD_NOW | os.RTLD_LOCAL)
    return hasattr(lib, name)


def test_find_equals_dlsym(fx):
    emu = FL.EmuResolver()
    want = {"plain": True, "default_v1": True, "hidden_v1": False, "local_all": False, "weak": True, "object": True,
            "via_needed": True, "outside_closure": False, "hash_gnu": True, "hash_sysv": True, "hash_both": True}
    sib = os.path.join(os.path.dirname(fx["plain"][0]), "libsibling.so")
    files = sorted({p for m, deps_, _ in fx.values() for p in [m] + deps_} | {sib})
    blobs = []
    for p in files:
        with open(p, "rb") as f:
            blobs.append(f.read())
    ids = {p: got[0] for p, got in zip(files, emu.index_blobs(blobs))}
    queries, scope = [], []
    for label in sorted(fx):
        m, more, name = fx[label]
        queries.append((len(scope), 1 + len(more), name.encode()))
        scope += [ids[m]] + [ids[p] for p in more]
    got = dict(zip(sorted(fx), emu.find(queries, scope)))
    for label in sorted(fx):
        m, more, name = fx[label]
        real = dlsym_finds(m, name)
        assert real == want[label], label
        assert (got[label][0] is not None) == real, label
        if real:
            assert got[label][0] == ids[more[0] if label == "via_needed" else m], label
    # the object the name resolves to and what the record says of it
    obj = got["object"]
    assert obj[2] & 0xf == 1 and obj[2] >> 4 == 1  # STT_OBJECT, STB_GLOBAL
    assert got["weak"][2] >> 4 == 2 and got["default_v1"][4] == 2  # STB_WEAK; versym index 2 (V1, the default)
    # an empty scope finds nothing
    assert emu.find([(0, 0, b"PyInit_plain")], []) == [(None, 0, 0, 0, 0)]


def test_queries_outside_the_pool_or_scope_are_refused(fx):
    emu = FL.EmuResolver()
    with open(fx["plain"][0], "rb") as f:
        emu.index_blobs([f.read()])
    cq, pool, found = deps.find_arrays([(0, 1, b"PyInit_plain")])
    cs = (ctypes.c_uint32 * 1)(0)
    assert emu.lib.lb2emu_syms_find(emu.h, cq, 1, cs, 1, pool, len(pool), found) == 0 and found[0].obj == 0
    cq[0].name_len = len(pool) + 1
    assert emu.lib.lb2emu_syms_find(emu.h, cq, 1, cs, 1, pool, len(pool), found) == -2
    cq[0].name_len, cq[0].scope_len = len(pool), 2
    assert emu.lib.lb2emu_syms_find(emu.h, cq, 1, cs, 1, pool, len(pool), found) == -2
    cs[0] = 5
    cq[0].scope_len = 1
    assert emu.lib.lb2emu_syms_find(emu.h, cq, 1, cs, 1, pool, len(pool), found) == -2


def test_asan_find_over_mutants_and_pool_edges(fx, tmp_path):
    exe = FL.asan_exe(str(tmp_path))
    small = D.linked_corpus(str(tmp_path / "linked"))
    names = "PyInit_plain,,v1,a_val,PyInit_h_gnu,x" + "y" * 300
    for bi, base in enumerate([fx["plain"][0], fx["default_v1"][0], small["libv.so"], small["libuser_gold.so"]]):
        with open(base, "rb") as f:
            data = f.read()
        files = []
        for j, (_, m) in enumerate(symbol_mutants(data, 100 + bi)):
            p = tmp_path / ("m%d_%d" % (bi, j))
            p.write_bytes(m)
            files.append(str(p))
        r = subprocess.run([exe] + files, capture_output=True, text=True, env=dict(os.environ, LB2EMU_FIND=names))
        assert r.returncode == 0, (base, r.stderr[-3000:])
        assert sum(1 for line in r.stdout.splitlines() if line.startswith("find ")) == 6
    # names at the pool's edges: the first, the last, an empty one, and one that is the whole pool
    plain = fx["plain"][0]
    for names in ("PyInit_plain", ",PyInit_plain", "PyInit_plain,", "a,PyInit_plain", ""):
        r = subprocess.run([exe, plain, small["libv.so"]], capture_output=True, text=True,
                           env=dict(os.environ, LB2EMU_FIND=names))
        assert r.returncode == 0, (names, r.stderr[-3000:])
        finds = [line.split()[1] for line in r.stdout.splitlines() if line.startswith("find ")]
        assert finds == ["0" if n == "PyInit_plain" else "-1" for n in names.split(",")], (names, finds)
