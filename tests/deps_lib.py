"""Shared by the dependency-check tests: the CPU emulator of the PRODUCT's dynamic-section parse
(tests/emu/deps_emu.cpp over lambdipy_b200/csrc/elf_deps.cuh, built with g++, plain or under
-fsanitize=address,undefined), `readelf -dVW` read into the same records, and the corpus of objects they are compared
on: the golden inputs, the elf_fixtures variants, libraries linked here with RPATH / RUNPATH / version scripts / gold,
and numpy's and scipy's shared objects.  Test harness only: never used by the package."""
import ctypes
import os
import re
import subprocess

import elf_fixtures as F
from lambdipy_b200 import _native as N

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "deps_emu.cpp")
HDR = os.path.join(ROOT, "lambdipy_b200", "csrc", "elf_deps.cuh")
FLAG_NAMES = {"BASE": 1, "WEAK": 2, "INFO": 4}


def _build(outdir):
    lib = os.path.join(outdir, "_build_deps_emu.so")
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in (SRC, HDR)):
        subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-o", lib, SRC], check=True)
    return lib


class Emu:
    """parse([bytes]) -> [(status, machine, [(kind, flags, ref, name)])], the records as lb2_elf_deps returns them"""

    def __init__(self, outdir=os.path.join(HERE, "emu")):
        self.lib = ctypes.CDLL(_build(outdir))
        vp, u64p = ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)
        self.lib.lb2emu_elf_deps.argtypes = [ctypes.POINTER(ctypes.c_void_p), u64p, ctypes.c_uint32,
                                             ctypes.POINTER(N.ElfObject), ctypes.POINTER(vp), u64p, ctypes.POINTER(vp), u64p]
        self.lib.lb2emu_elf_deps.restype = ctypes.c_int
        self.lib.lb2emu_free.argtypes = [vp]

    def parse(self, blobs):
        n = len(blobs)
        bufs = [ctypes.create_string_buffer(b, len(b)) for b in blobs]  # exactly len(b) bytes: no NUL after
        ptrs = (ctypes.c_void_p * max(n, 1))(*[ctypes.addressof(b) for b in bufs])
        sizes = (ctypes.c_uint64 * max(n, 1))(*[len(b) for b in blobs])
        objs = (N.ElfObject * max(n, 1))()
        rec, pool, nr, npool = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_uint64()
        assert self.lib.lb2emu_elf_deps(ptrs, sizes, n, objs, ctypes.byref(rec), ctypes.byref(nr), ctypes.byref(pool),
                                        ctypes.byref(npool)) == 0, "the count and write passes disagree"
        recs = (N.ElfRecord * nr.value).from_address(rec.value) if nr.value else []
        pool_b = ctypes.string_at(pool.value, npool.value) if npool.value else b""
        out = decode(objs[:n], recs, pool_b)
        self.lib.lb2emu_free(rec)
        self.lib.lb2emu_free(pool)
        return out


def decode(objs, recs, pool):
    """lb2_elf_object / lb2_elf_record arrays and the pool -> [(status, machine, [(kind, flags, ref, name)])]"""
    out = []
    for o in objs:
        rs = []
        for r in recs[o.first_record:o.first_record + o.n_records]:
            assert pool[r.off + r.len] == 0
            rs.append((r.kind, r.flags, r.ref, pool[r.off:r.off + r.len].decode("utf-8", "surrogateescape")))
        out.append((o.status, o.machine, rs))
    return out


def asan_exe(outdir):
    """the emulator as a program built under -fsanitize=address,undefined (deps_emu.cpp's main): `exe FILE...` parses
    the files, each in a buffer of exactly its size, and prints "status records pool_bytes" per file; any sanitizer
    report ends it with a non-zero status"""
    exe = os.path.join(outdir, "deps_emu_asan")
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in (SRC, HDR)):
        subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-Wall", "-Werror", "-DLB2EMU_MAIN", "-fsanitize=address,undefined",
                        "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe, SRC], check=True)
    return exe


_DYN = re.compile(r"^\s*0x[0-9a-f]+ \((NEEDED|SONAME|RPATH|RUNPATH)\)\s+\S.*?: \[(.*)\]$")
_VN_FILE = re.compile(r"^\s*[0-9a-fx]+: Version: \d+\s+File: (.*?)\s+Cnt: \d+$")
_VN_NAME = re.compile(r"^\s*0x[0-9a-f]+:\s+Name: (.*?)\s+Flags: (.*?)\s+Version: \d+$")
_VD = re.compile(r"^\s*[0-9a-fx]+: Rev: \d+\s+Flags: (.*?)\s+Index: \d+\s+Cnt: (\d+)\s+Name: (.*)$")
_KIND = {"NEEDED": N.ELF_REC_NEEDED, "SONAME": N.ELF_REC_SONAME, "RPATH": N.ELF_REC_RPATH, "RUNPATH": N.ELF_REC_RUNPATH}


def _flags(s):
    if s == "none":
        return 0
    names = [f.strip() for f in s.split("|")]
    return sum(FLAG_NAMES[f] for f in names) if all(f in FLAG_NAMES for f in names) else -1  # -1: readelf's <unknown>


def readelf(path):
    """(records in lb2_elf_deps' order, whether readelf complained) from `readelf -dVW path`"""
    r = subprocess.run(["readelf", "-dVW", path], capture_output=True)
    text = r.stdout.decode("utf-8", "surrogateescape")
    complained = r.returncode != 0 or b"Error" in r.stderr or b"Warning" in r.stderr or b"<corrupt" in r.stdout
    dyn, vn, vd, section = [], [], [], None
    for line in text.splitlines():
        if line.startswith("Version needs section"):
            section = "vn"
        elif line.startswith("Version definition section"):
            section = "vd"
        elif line.startswith("Version symbols section") or line.startswith("Dynamic section"):
            section = None
        m = _DYN.match(line)
        if m:
            dyn.append((_KIND[m.group(1)], 0, 0, m.group(2)))
            continue
        if section == "vn":
            m = _VN_FILE.match(line)
            if m:
                vn.append([m.group(1), []])
                continue
            m = _VN_NAME.match(line)
            if m:
                vn[-1][1].append((m.group(1), _flags(m.group(2))))
        elif section == "vd":
            m = _VD.match(line)
            if m and int(m.group(2)):
                vd.append((N.ELF_REC_VERDEF, _flags(m.group(1)), 0, m.group(3)))
    recs = list(dyn)
    for file, names in vn:
        at = len(recs)
        recs.append((N.ELF_REC_VERNEED_FILE, 0, 0, file))
        recs += [(N.ELF_REC_VERNEED_VERSION, fl, at, name) for name, fl in names]
    return recs + vd, complained


LIB_A = "int a_val(void) { return 1; }\n"
LIB_V = "int v1(void) { return 1; }\nint v2(void) { return 2; }\n"
VSCRIPT = "V1 { global: v1; local: *; };\nV2 { global: v2; } V1;\n"
USER = "int v1(void); int v2(void); int a_val(void);\nint use(void) { return v1() + v2() + a_val(); }\n"


def linked_corpus(outdir):
    """Libraries linked here: {name: path}.  RUNPATH (--enable-new-dtags) and RPATH (--disable-new-dtags) users of
    liba, a --version-script library (VERDEF) and its user (VERNEED on it), and gold-linked ones."""
    os.makedirs(outdir, exist_ok=True)
    def src(name, text):
        p = os.path.join(outdir, name)
        with open(p, "w") as f:
            f.write(text)
        return p
    a, v, vs, u = src("a.c", LIB_A), src("v.c", LIB_V), src("v.map", VSCRIPT), src("user.c", USER)
    out = {}
    def cc(name, args):
        p = os.path.join(outdir, name)
        r = subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-o", p] + args, capture_output=True)
        if r.returncode == 0:
            out[name] = p
    cc("liba.so", [a, "-Wl,-soname,liba.so.1"])
    cc("libv.so", [v, "-Wl,--version-script=" + vs, "-Wl,-soname,libv.so"])
    for dt, flag in (("runpath", "--enable-new-dtags"), ("rpath", "--disable-new-dtags")):
        cc("libuser_%s.so" % dt, [u, "-L" + outdir, "-Wl,-rpath,$ORIGIN:/opt/lib", "-Wl," + flag, "-lv", "-la"])
    cc("libv_gold.so", [v, "-fuse-ld=gold", "-Wl,--version-script=" + vs, "-Wl,-soname,libv.so"])
    cc("libuser_gold.so", [u, "-fuse-ld=gold", "-L" + outdir, "-Wl,-rpath,$ORIGIN", "-lv", "-la"])
    return out


def site_objects():
    """numpy's and scipy's shared objects and their .libs (present on every machine this suite runs on)"""
    sp = F.site_packages()
    files = []
    for r in ("numpy", "scipy", "numpy.libs", "scipy.libs"):
        for d, _, fs in os.walk(os.path.join(sp, r)):
            for f in fs:
                p = os.path.join(d, f)
                if ".so" in f and not os.path.islink(p):
                    with open(p, "rb") as fh:
                        if fh.read(4) == b"\x7fELF":
                            files.append(p)
    return sorted(files)


def corpus(tmp):
    """{label: path} of every object the records are checked on"""
    out = {}
    gdir = os.path.join(HERE, "golden")
    for f in sorted(os.listdir(gdir)):
        if f.endswith(".in.bin"):
            out["golden/" + f] = os.path.join(gdir, f)
    for name, p in F.build_variants(os.path.join(tmp, "variants")).items():
        out["variant/" + name] = p
    for name, p in linked_corpus(os.path.join(tmp, "linked")).items():
        out["linked/" + name] = p
    sp = F.site_packages()
    for p in site_objects():
        out["site/" + os.path.relpath(p, sp)] = p
    return out
