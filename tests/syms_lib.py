"""Shared by the symbol-check tests: the CPU emulator of the PRODUCT's symbol index and lookup
(tests/emu/syms_emu.cpp over lambdipy_b200/csrc/elf_syms.cuh, built with g++, plain or under
-fsanitize=address,undefined), a stand-in for GpuSymbolResolver over it, and `readelf -rsW` read into the reference
lists the index must produce.  Test harness only: never used by the package."""
import ctypes
import os
import re
import subprocess

from lambdipy_b200 import _native as N

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "syms_emu.cpp")
HDRS = [os.path.join(ROOT, "lambdipy_b200", "csrc", h) for h in ("elf_syms.cuh", "elf_deps.cuh")]


def _stale(out):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in [SRC] + HDRS)


def _build(outdir):
    lib = os.path.join(outdir, "_build_syms_emu.so")
    if _stale(lib):
        subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-o", lib, SRC], check=True)
    return lib


def asan_exe(outdir):
    """syms_emu.cpp's main under -fsanitize=address,undefined: `exe FILE...` indexes the files (each in a buffer of
    exactly its size), resolves every object's references in the scope of all of them and prints "status symbols
    references misses" per file"""
    exe = os.path.join(outdir, "syms_emu_asan")
    if _stale(exe):
        subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-Wall", "-Werror", "-DLB2EMU_MAIN", "-fsanitize=address,undefined",
                        "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe, SRC], check=True)
    return exe


class _Lib:
    _lib = None

    @classmethod
    def get(cls):
        if cls._lib is None:
            lib = ctypes.CDLL(_build(os.path.join(HERE, "emu")))
            vp, u32p, u64p = ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint64)
            lib.lb2emu_syms_create.restype = vp
            lib.lb2emu_syms_destroy.argtypes = [vp]
            lib.lb2emu_syms_index.argtypes = [vp, ctypes.POINTER(vp), u64p, ctypes.c_uint32, u32p, ctypes.POINTER(N.SymObject)]
            lib.lb2emu_syms_refs.argtypes = [vp, ctypes.c_uint32]
            lib.lb2emu_syms_refs.restype = ctypes.POINTER(N.SymRef)
            lib.lb2emu_syms_resolve.argtypes = [vp, ctypes.POINTER(N.SymJob), ctypes.c_uint32, u32p,
                                                ctypes.POINTER(ctypes.c_uint8), u32p, ctypes.POINTER(N.SymMiss),
                                                ctypes.c_uint32, u32p, u64p]
            lib.lb2emu_syms_name.argtypes = [vp, ctypes.POINTER(N.SymJob), N.SymMiss, ctypes.c_char_p, ctypes.c_uint64]
            lib.lb2emu_syms_name.restype = ctypes.c_uint64
            cls._lib = lib
        return cls._lib


class EmuResolver:
    """GpuSymbolResolver's interface over the emulator.  mem: the tests' fake device memory (get((addr, n)) -> bytes),
    or None for index_blobs only."""

    def __init__(self, mem=None):
        self.lib, self.mem = _Lib.get(), mem
        self.h = self.lib.lb2emu_syms_create()
        self.uploaded = self.downloaded = 0
        self.objects = []

    def index_blobs(self, blobs):
        n = len(blobs)
        bufs = [ctypes.create_string_buffer(b, len(b)) for b in blobs]
        ptrs = (ctypes.c_void_p * max(n, 1))(*[ctypes.addressof(b) for b in bufs])
        sizes = (ctypes.c_uint64 * max(n, 1))(*[len(b) for b in blobs])
        ids, objs = (ctypes.c_uint32 * max(n, 1))(), (N.SymObject * max(n, 1))()
        self.lib.lb2emu_syms_index(self.h, ptrs, sizes, n, ids, objs)
        self.objects += [objs[i] for i in range(n)]
        return [(ids[i], objs[i].status, objs[i].nrefs) for i in range(n)]

    def index(self, refs):
        return self.index_blobs([self.mem.get(r) for r in refs])

    def refs(self, i):
        """object i's references: [(symbol index, name, versym index, weak)] (the names read back from the object)"""
        o = self.objects[i]
        p = self.lib.lb2emu_syms_refs(self.h, i)
        out = []
        for k in range(o.nrefs):
            r = p[k]
            name = ctypes.string_at(o.arena + tables_str(o) + r.name, r.name_len).decode("utf-8", "surrogateescape")
            out.append((r.sym, name, r.ver, r.weak, r.gnu, r.sysv))
        return out

    def resolve(self, jobs, scope, classes):
        nj = len(jobs)
        cj = (N.SymJob * max(nj, 1))(*[N.SymJob(o, off, ln, 0) for o, off, ln in jobs])
        cs = (ctypes.c_uint32 * max(len(scope), 1))(*scope)
        cc = (ctypes.c_uint8 * max(len(classes), 1))(*classes)
        counts = (ctypes.c_uint32 * max(3 * nj, 1))()
        cap = 1 << 20
        miss, nm, lookups = (N.SymMiss * cap)(), ctypes.c_uint32(), ctypes.c_uint64()
        self.lib.lb2emu_syms_resolve(self.h, cj, nj, cs, cc, counts, miss, cap, ctypes.byref(nm), ctypes.byref(lookups))
        self.lookups = lookups.value
        return [tuple(counts[3 * j:3 * j + 3]) for j in range(nj)], [(miss[i].job, miss[i].ref) for i in range(nm.value)]

    def names(self, jobs, misses):
        cj = (N.SymJob * max(len(jobs), 1))(*[N.SymJob(o, off, ln, 0) for o, off, ln in jobs])
        out = []
        for j, r in misses:
            buf = ctypes.create_string_buffer(1 << 16)
            self.lib.lb2emu_syms_name(self.h, cj, N.SymMiss(j, r), buf, len(buf))
            out.append(tuple(x.decode("utf-8", "surrogateescape") for x in buf.raw.split(b"\0", 3)[:3]))
        return out

    def stats(self):
        return {"index_ms": 0.0, "refs_ms": 0.0, "resolve_ms": 0.0, "lookups": getattr(self, "lookups", 0)}

    def close(self):
        if self.h:
            self.lib.lb2emu_syms_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()


def _al8(x):
    return (x + 7) & ~7


def tables_str(o):
    """elf_syms.cuh tables(o).str: where .dynstr lies in the object's arena block"""
    t = o.nsyms * 24
    t = _al8(t) + (o.nsyms * 2 if o.flags & 4 else 0)
    t = _al8(t) + o.hash_len
    t = _al8(t) + o.nver * 24
    t = _al8(t) + (o.nsyms + 31) // 32 * 4
    return _al8(t)


_SYM = re.compile(r"^\s*(\d+): ([0-9a-f]+)\s+\d+\s+(\w+)\s+(\w+)\s+(\w+)\s+(\S+)\s+(\S+)")


def readelf_refs(path):
    """{(name, version or "")} of the symbols relocations name that are UND and not LOCAL, from `readelf -rsW`
    (--dyn-syms for the symbol table, -r for the relocations' symbol indices shown by name)"""
    syms = subprocess.run(["readelf", "--dyn-syms", "-W", path], capture_output=True, text=True, errors="surrogateescape").stdout
    und = {}
    for line in syms.splitlines():
        m = _SYM.match(line)
        if m and m.group(6) == "UND" and m.group(4) != "LOCAL" and int(m.group(1)):
            full = m.group(7)
            name, _, ver = full.partition("@")
            und[(name, ver.split(" ")[0].lstrip("@"))] = True
    rel = subprocess.run(["readelf", "-rW", path], capture_output=True, text=True, errors="surrogateescape").stdout
    out = set()
    for line in rel.splitlines():
        parts = line.split()
        if len(parts) >= 5 and re.fullmatch(r"[0-9a-f]{16}", parts[0]) and re.fullmatch(r"[0-9a-f]{16}", parts[3]):
            name, _, ver = parts[4].partition("@")
            key = (name, ver.lstrip("@"))
            if key in und:
                out.add(key)
    return out
