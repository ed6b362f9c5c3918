"""CPU checks of the zip reader's member-table pipeline without a GPU: the product's ifl::Batch and decoding core
(lambdipy_b200/csrc/inflate_core.cuh) are compiled with g++ into a harness (tests/emu/unzip_emu.cpp) that runs them in
the order lb2_unzip_run launches them.  Many members share one buffer, separated by filler bytes, so every test also
checks that no decoder reads or resolves outside its own member."""
import ctypes
import os
import random
import subprocess
import zlib

import pytest

import deflate_ref as R
import inflate_streams as IS

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "unzip_emu.cpp")
LIB = os.path.join(HERE, "emu", "_build_unzip_emu.so")
DEPS = [SRC, os.path.join(ROOT, "lambdipy_b200", "csrc", "inflate_core.cuh")]
OK, BAD_DATA, WRONG_SIZE = 0, 1, 2


class UnzipEmu:
    def __init__(self):
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
            subprocess.run(["g++", "-std=c++17", "-O2", "-g", "-shared", "-fPIC", "-Wall", "-o", LIB, SRC], check=True)
        lib = self.lib = ctypes.CDLL(LIB)
        u64, u64p, vp = ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p
        lib.lb2emu_unzip.argtypes = [ctypes.c_char_p, u64, u64p, ctypes.c_uint32, u64, ctypes.POINTER(vp), u64p, u64p,
                                     ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_uint32)]
        lib.lb2emu_unzip.restype = ctypes.c_int
        lib.lb2emu_free.argtypes = [vp]

    def run(self, members, span, seed=0):
        """members: [(body, size, method)] -> ([(status, bytes)], stats).  Bodies are laid out with random filler
        (as local headers and other members' bodies would be) between them."""
        rng = random.Random(seed)
        buf, rows = bytearray(rng.randbytes(rng.randrange(64))), []
        for body, size, method in members:
            rows += [len(buf), len(body), size, method]
            buf += body + rng.randbytes(rng.randrange(1, 64))
        k = len(members)
        out, n = ctypes.c_void_p(), ctypes.c_uint64()
        offs, status, st = (ctypes.c_uint64 * max(k, 1))(), (ctypes.c_int32 * max(k, 1))(), (ctypes.c_uint32 * 6)()
        rc = self.lib.lb2emu_unzip(bytes(buf), len(buf), (ctypes.c_uint64 * max(len(rows), 1))(*rows), k, span,
                                   ctypes.byref(out), ctypes.byref(n), offs, status, st)
        assert rc == 0
        data = ctypes.string_at(out.value, n.value) if n.value else b""
        self.lib.lb2emu_free(out)
        res = [(status[i], data[offs[i]:offs[i] + m[1]]) for i, m in enumerate(members)]
        return res, dict(zip(("n_stored", "n_small", "n_large", "n_spans", "n_rounds", "n_rejected"), list(st)))


def zlib_or_none(body):
    try:
        return zlib.decompress(body, -15)
    except zlib.error:
        return None


@pytest.fixture(scope="module")
def emu():
    return UnzipEmu()


@pytest.fixture(scope="module")
def zlib_members():
    """zlib levels 1/6/9 and 0, its strategies and flush modes, edge sizes, plus STORED and empty members"""
    members = [(name, body, data, 8) for name, body, data in IS.matrix(96 << 10)]
    for n in (0, 1, 17, 5000, 70000):
        data = IS.text(n, seed=n + 3)
        members.append(("stored-%d" % n, data, data, 0))
    members.append(("empty-deflate", zlib.compress(b"", 6)[2:-4], b"", 8))
    members.append(("empty-final-block", b"\x03\x00", b"", 8))
    return members


@pytest.mark.parametrize("span", [1024, 3000, 8192])
def test_members_equal_zlib(emu, zlib_members, span):
    res, st = emu.run([(body, len(data), method) for _, body, data, method in zlib_members], span, seed=span)
    for (name, _, data, _), (status, got) in zip(zlib_members, res):
        assert status == OK, (name, status)
        assert got == data, name
    assert st["n_stored"] == 5 and st["n_small"] > 0 and st["n_large"] > 0, st
    assert st["n_spans"] > st["n_large"], st  # the larger members really were cut into spans


@pytest.mark.parametrize("span", [1024, 2048, 8192])
def test_crafted_corpus_as_members(emu, span):
    corpus = R.crafted(deltas=(0,), phases=(0, 3, 7)) + R.crafted(deltas=(-3, 5), phases=(5,))[:-len(R.unplaced())]
    want = [zlib_or_none(body) for _, body in corpus]
    members = [(body, len(w) if w is not None else 100, 8) for (_, body), w in zip(corpus, want)]
    res, _ = emu.run(members, span, seed=span + 1)
    n_refused = 0
    for (name, _), w, (status, got) in zip(corpus, want, res):
        if w is None:
            n_refused += 1
            assert status != OK, name
        else:
            assert status == OK and got == w, (name, status)
    assert n_refused > 10


def back_past_start():
    """a STORED block of 4000 bytes, then a dynamic block whose first match reaches 5000 bytes back"""
    s = R.Stream()
    s.stored(R._bytes(4000, 5))
    s.dynamic([(6, 5000)] + R._lit_text(40, 6), final=True)
    return s.body()


@pytest.mark.parametrize("span", [1024, 2048])
def test_match_back_past_member_start_is_refused(emu, span):
    bad = back_past_start()
    assert zlib_or_none(bad) is None
    before = IS.text(40000, seed=11)  # 32 KB of real output just before the bad member's output
    after = IS.so_bytes(50000)
    members = [(IS.deflate(before, 9), len(before), 8), (bad, 4046, 8), (IS.deflate(after, 6), len(after), 8)]
    res, st = emu.run(members, span)
    assert st["n_large"] == 3, st
    assert res[0] == (OK, before)
    assert res[1][0] == BAD_DATA
    assert res[2] == (OK, after)


@pytest.mark.parametrize("span", [1024, 1 << 20])
def test_wrong_sizes_and_truncation(emu, span):
    data = IS.text(30000, seed=2)
    body = IS.deflate(data, 6)
    members = [(body, len(data), 8), (body, len(data) - 1, 8), (body, len(data) + 1, 8), (body[:-3], len(data), 8),
               (data, len(data) - 1, 0), (body, len(data), 8)]
    res, _ = emu.run(members, span)
    assert [r[0] for r in res] == [OK, WRONG_SIZE, WRONG_SIZE, BAD_DATA, WRONG_SIZE, OK]
    assert res[0][1] == res[5][1] == data
