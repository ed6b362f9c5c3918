"""CPU checks of the PRODUCT's seek-table path (ifl::Table and the exact-stop mode of decode_span in
lambdipy_b200/csrc/inflate_core.cuh) without a GPU: the core is compiled with g++ into a harness (tests/emu/seek_emu.cpp)
that decodes one exact-stop span per entry, accepts or refuses the table as lb2_inflate_run_table does, and falls back
to the search pipeline.  Honest tables over zlib streams flushed at 64 KB and at odd offsets (sync and full flushes,
fixed-Huffman and stored chunks, levels 1/6/9) are accepted and give zlib's bytes; tampered tables are refused and
still give zlib's bytes."""
import ctypes
import os
import subprocess
import zlib

import pytest

import seek_streams as SS

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "seek_emu.cpp")
LIB = os.path.join(HERE, "emu", "_build_seek_emu.so")
DEPS = [SRC, os.path.join(HERE, "emu", "inflate_emu.cpp"), os.path.join(ROOT, "lambdipy_b200", "csrc", "inflate_core.cuh")]


class Emu:
    def __init__(self):
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
            subprocess.run(["g++", "-std=c++17", "-O2", "-g", "-shared", "-fPIC", "-Wall", "-o", LIB, SRC], check=True)
        lib = self.lib = ctypes.CDLL(LIB)
        u64, u64p, vp = ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p
        lib.lb2emu_table_inflate.argtypes = [ctypes.c_char_p, u64, u64p, ctypes.c_uint32, u64, ctypes.POINTER(vp), u64p,
                                             u64p, ctypes.POINTER(ctypes.c_int)]
        lib.lb2emu_table_inflate.restype = ctypes.c_int
        lib.lb2emu_inflate.argtypes = [ctypes.c_char_p, u64, u64, ctypes.POINTER(vp), u64p,
                                       ctypes.POINTER(ctypes.c_uint32), u64p]
        lib.lb2emu_inflate.restype = ctypes.c_int
        lib.lb2emu_free.argtypes = [vp]

    def _take(self, rc, out, n):
        if rc:
            return None
        data = ctypes.string_at(out.value, n.value) if n.value else b""
        self.lib.lb2emu_free(out)
        return data

    def table(self, body, entries, span=128 << 10):
        """-> (status, bytes | None, in_bytes, table used)"""
        flat = (ctypes.c_uint64 * max(2 * len(entries), 1))(*[v for e in entries for v in e])
        out, n, ib, used = ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int()
        rc = self.lib.lb2emu_table_inflate(body, len(body), flat, len(entries), span, ctypes.byref(out), ctypes.byref(n),
                                           ctypes.byref(ib), ctypes.byref(used))
        return rc, self._take(rc, out, n), ib.value, used.value

    def search(self, body, span=128 << 10):
        out, n, ib = ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_uint64()
        st = (ctypes.c_uint32 * 4)()
        rc = self.lib.lb2emu_inflate(body, len(body), span, ctypes.byref(out), ctypes.byref(n), st, ctypes.byref(ib))
        return rc, self._take(rc, out, n), ib.value


@pytest.fixture(scope="module")
def emu():
    return Emu()


@pytest.fixture(scope="module")
def streams():
    return SS.matrix()


def test_honest_tables_decode_as_zlib(emu, streams):
    for name, body, data, entries in streams:
        assert zlib.decompress(body, -15) == data, name
        rc, out, ib, used = emu.table(body + b"trailer!", entries)
        assert (rc, used, ib) == (0, 1, len(body)), name
        assert out == data, name


def test_tampered_tables_fall_back_to_the_search(emu, streams):
    refused = 0
    for name, body, data, entries in streams:
        want = emu.search(body + bytes(8))
        assert want[:2] == (0, data), name
        for how, t in SS.tampered(entries):
            rc, out, ib, used = emu.table(body + bytes(8), t)
            assert (rc, out, ib) == want, (name, how)
            if t != entries:
                assert used == 0, (name, how)
                refused += 1
    assert refused > 100


def test_a_final_block_inside_the_table(emu, streams):
    """a stream whose first run already ends the stream: the table claims more after it"""
    _, body, data, entries = streams[0]
    head = zlib.compressobj(6, zlib.DEFLATED, -15)
    first = head.compress(data[:SS.CHUNK]) + head.flush()
    stream = first + body
    t = [(len(first), SS.CHUNK)] + entries
    rc, out, ib, used = emu.table(stream, t)
    assert (rc, out, ib, used) == (0, data[:SS.CHUNK], len(first), 0)


def test_table_granularity_does_not_matter(emu, streams):
    """any grouping of whole chunks is a valid table: runs of 3 and the whole stream in two entries"""
    for name, body, data, entries in streams:
        for t in (_runs(entries, 3), [(sum(c for c, _ in entries[:-1]), sum(u for _, u in entries[:-1])), entries[-1]]):
            rc, out, ib, used = emu.table(body, t)
            assert (rc, out, used) == (0, data, 1), name


def _runs(entries, k):
    return [(sum(c for c, _ in entries[i:i + k]), sum(u for _, u in entries[i:i + k])) for i in range(0, len(entries), k)]
