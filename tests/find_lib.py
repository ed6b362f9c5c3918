"""Shared by the import-check tests: the CPU emulator of the PRODUCT's dlsym-style lookup behind lb2_syms_find
(tests/emu/syms_find_emu.cpp over lambdipy_b200/csrc/elf_syms.cuh and the resolver emulator of syms_emu.cpp, built
with g++, plain or under -fsanitize=address,undefined) and a stand-in for GpuSymbolResolver that adds find() to
syms_lib.EmuResolver.  Test harness only: never used by the package."""
import ctypes
import os
import subprocess

import syms_lib as S
from lambdipy_b200 import _native as N
from lambdipy_b200 import deps

SRC = os.path.join(S.HERE, "emu", "syms_find_emu.cpp")
DEPS = [SRC, S.SRC] + S.HDRS


def _stale(out):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in DEPS)


def asan_exe(outdir):
    """syms_find_emu.cpp's main under -fsanitize=address,undefined: `LB2EMU_FIND=a,b exe FILE...` indexes the files
    (each in a buffer of exactly its size), prints "status symbols" per file, then looks each name up in the scope of
    all of them and prints "find OBJECT SYMBOL" per name (OBJECT -1: none)"""
    exe = os.path.join(outdir, "syms_find_emu_asan")
    if _stale(exe):
        subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-Wall", "-Werror", "-DLB2EMU_FIND_MAIN",
                        "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                        SRC], check=True)
    return exe


_LIB = []


def _lib():
    """the emulator library, with syms_lib's argument types for the functions it shares with syms_emu.cpp"""
    if not _LIB:
        out = os.path.join(S.HERE, "emu", "_build_syms_find_emu.so")
        if _stale(out):
            subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-Wall", "-Werror", "-o", out, SRC],
                           check=True)
        lib, base = ctypes.CDLL(out), S._Lib.get()
        for name in ("lb2emu_syms_create", "lb2emu_syms_destroy", "lb2emu_syms_index", "lb2emu_syms_refs",
                     "lb2emu_syms_resolve", "lb2emu_syms_name"):
            f, g = getattr(lib, name), getattr(base, name)
            f.argtypes, f.restype = g.argtypes, g.restype
        lib.lb2emu_syms_find.argtypes = [ctypes.c_void_p, ctypes.POINTER(N.SymQuery), ctypes.c_uint32,
                                         ctypes.POINTER(ctypes.c_uint32), ctypes.c_uint32, ctypes.c_char_p,
                                         ctypes.c_uint64, ctypes.POINTER(N.SymFound)]
        _LIB.append(lib)
    return _LIB[0]


class EmuResolver(S.EmuResolver):
    """GpuSymbolResolver's interface over the emulator, find() included"""

    def __init__(self, mem=None):
        self.lib, self.mem = _lib(), mem
        self.h = self.lib.lb2emu_syms_create()
        self.uploaded = self.downloaded = 0
        self.objects = []
        self.finds = 0

    def find(self, queries, scope):
        """GpuSymbolResolver.find over the emulator"""
        cq, pool, found = deps.find_arrays(queries)
        cs = (ctypes.c_uint32 * max(len(scope), 1))(*scope)
        if self.lib.lb2emu_syms_find(self.h, cq, len(queries), cs, len(scope), pool, len(pool), found):
            raise ValueError("lb2emu_syms_find: a query outside the scope array or the name pool")
        self.finds += len(queries)
        return deps.found_records(found, len(queries))

    def stats(self):
        return dict(super().stats(), find_ms=0.0, find_queries=self.finds)
