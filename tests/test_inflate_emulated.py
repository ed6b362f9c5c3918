"""CPU checks of the PRODUCT's inflate core (lambdipy_b200/csrc/inflate_core.cuh) without a GPU: the core is compiled
with g++ into a harness (tests/emu/inflate_emu.cpp) that runs the candidate search, the count rounds and chain, the
decode pass and the resolve steps in the CUDA pipeline's order.  The GPU tests remain the check of the compiled
library; these let the decoder logic be developed and checked on a machine without one."""
import ctypes
import os
import subprocess
import zlib

import pytest

import inflate_streams as IS

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "inflate_emu.cpp")
LIB = os.path.join(HERE, "emu", "_build_inflate_emu.so")
DEPS = [SRC, os.path.join(ROOT, "lambdipy_b200", "csrc", "inflate_core.cuh")]


class Emu:
    def __init__(self):
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
            subprocess.run(["g++", "-std=c++17", "-O2", "-g", "-shared", "-fPIC", "-Wall", "-o", LIB, SRC], check=True)
        lib = self.lib = ctypes.CDLL(LIB)
        u64, u64p, vp = ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p
        lib.lb2emu_inflate.argtypes = [ctypes.c_char_p, u64, u64, ctypes.POINTER(vp), u64p, ctypes.POINTER(ctypes.c_uint32), u64p]
        lib.lb2emu_inflate.restype = ctypes.c_int
        lib.lb2emu_block_keys.argtypes = [ctypes.c_char_p, u64, u64p, u64]
        lib.lb2emu_block_keys.restype = ctypes.c_int64
        lib.lb2emu_candidate.argtypes = [ctypes.c_char_p, u64, u64]
        lib.lb2emu_candidate.restype = u64
        lib.lb2emu_free.argtypes = [vp]

    def inflate(self, body, span):
        """-> (status, bytes | None, stats dict)"""
        out, n, ib = ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_uint64()
        st = (ctypes.c_uint32 * 4)()
        rc = self.lib.lb2emu_inflate(body, len(body), span, ctypes.byref(out), ctypes.byref(n), st, ctypes.byref(ib))
        stats = dict(zip(("n_spans", "n_rounds", "n_rejected", "n_absorbed"), list(st)), in_bytes=ib.value)
        if rc:
            return rc, None, stats
        data = ctypes.string_at(out.value, n.value) if n.value else b""
        self.lib.lb2emu_free(out)
        return 0, data, stats

    def block_keys(self, body):
        cap = len(body) + 16
        keys = (ctypes.c_uint64 * cap)()
        k = self.lib.lb2emu_block_keys(body, len(body), keys, cap)
        assert k >= 0, k
        return list(keys[:k])

    def candidate(self, body, bit):
        return self.lib.lb2emu_candidate(body, len(body), bit)


@pytest.fixture(scope="module")
def emu():
    return Emu()


@pytest.fixture(scope="module")
def streams():
    return IS.matrix(256 << 10)


def test_filter_passes_every_true_block_start(emu, streams):
    n_dyn = n_stored = 0
    for name, body, _ in streams:
        for key in emu.block_keys(body):
            bit, stored, bfinal = key >> 2, (key >> 1) & 1, key & 1
            got = emu.candidate(body, bit)
            if stored:
                # A final stored block's BFINAL bit cannot be told from the zero padding in front of LEN unless the
                # header sits right below it, and it has no next block to check; such a block is decoded by the span
                # before it (the chain rejects a wrong BFINAL, it never uses it).
                if bfinal:
                    continue
                n_stored += 1
                assert got == key, (name, bit)
            else:
                n_dyn += 1
                assert got == key, (name, bit)
    assert n_dyn > 200 and n_stored > 100, (n_dyn, n_stored)


@pytest.mark.parametrize("span", [1024, 3000, 8192])
def test_pipeline_equals_zlib(emu, streams, span):
    for name, body, data in streams:
        st, got, stats = emu.inflate(body, span)
        assert st == 0, (name, st, stats)
        assert got == data, name
        assert stats["in_bytes"] == len(body), (name, stats)


def test_pipeline_runs_in_parallel_and_rejects(emu):
    data = IS.so_bytes(4 << 20)
    body = IS.deflate(data, 9)
    span = 64 << 10   # a few zlib-9 blocks per span
    st, got, stats = emu.inflate(body, span)
    assert st == 0 and got == data
    nominal = (len(body) + span - 1) // span
    assert stats["n_spans"] >= nominal * 0.8, stats
    # outer stored blocks carrying inner DEFLATE streams: the filter finds inner headers, the chain rejects them
    inner = b"".join(zlib.compress(IS.so_bytes(256 << 10)[k::3], 9) for k in range(3))
    body = IS.deflate(inner, 0)
    st, got, stats = emu.inflate(body, 4096)
    assert st == 0 and got == inner
    assert stats["n_rejected"] > 0, stats


def test_trailing_bytes_and_corrupt_input(emu):
    data = IS.text(300 << 10)
    body = IS.deflate(data, 9)
    st, got, stats = emu.inflate(body + b"\x12\x34\x56\x78" * 2 + body, 2048)   # trailer and a second stream after it
    assert st == 0 and got == data and stats["in_bytes"] == len(body)
    for cut in (1, len(body) // 2, len(body) - 1):
        st, got, _ = emu.inflate(body[:cut], 2048)
        assert st != 0 and got is None, cut
    for at in range(0, len(body), len(body) // 17):
        bad = bytearray(body)
        bad[at] ^= 0x5A
        st, got, _ = emu.inflate(bytes(bad), 2048)
        try:
            want = zlib.decompress(bytes(bad), -15)
        except zlib.error:
            want = None
        assert got is None or got == want, at   # never success with other bytes than zlib's
    assert emu.inflate(b"", 1024)[0] != 0
    assert emu.inflate(b"\x07", 1024)[0] != 0  # BTYPE 3
