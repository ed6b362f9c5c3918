"""CPU checks of the PRODUCT's optimal-parse core (lambdipy_b200/csrc/deflate_parse.cuh) without a GPU: the core is
compiled with g++ into a harness (tests/emu/parse_emu.cpp) that builds Pareto lists from hash-chain-ordered candidates,
relaxes one position at a time over 32 lanes, traces the path back and gathers its tokens, as the best-mode kernel
does.  On random bytes, runs, periodic data, text and a slice of a real shared object, with match candidates and bit
costs computed here:
* the Pareto lists are the ones a restatement in numpy keeps (longer and farther only, the K longest);
* the path cost equals a brute-force shortest path over the same edges, and the tokens cost exactly that;
* the tokens rebuild the input, and the same input gives the same tokens.
"""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "parse_emu.cpp")
LIB = os.path.join(HERE, "emu", "_build_parse_emu.so")
DEPS = [SRC, os.path.join(ROOT, "lambdipy_b200", "csrc", "deflate_parse.cuh")]
K = 8
LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
         6145, 8193, 12289, 16385, 24577]


@pytest.fixture(scope="module")
def emu():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-std=c++17", "-O2", "-g", "-shared", "-fPIC", "-Wall", "-o", LIB, SRC], check=True)
    lib = ctypes.CDLL(LIB)
    u64p = ctypes.POINTER(ctypes.c_uint64)
    lib.lb2emu_pareto.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p]
    lib.lb2emu_parse.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                 ctypes.c_void_p, ctypes.c_void_p, u64p]
    lib.lb2emu_parse.restype = ctypes.c_uint32
    return lib


def dist_sym(d):
    return max(i for i, b in enumerate(DBASE) if b <= d)


def len_sym(length):
    return 285 if length == 258 else 257 + max(i for i, b in enumerate(LBASE[:28]) if b <= length)


def candidates(data):
    """every (position, distance, length >= 3) of data, nearest distance first per position, as numpy arrays"""
    a = np.frombuffer(data, np.uint8)
    n = len(a)
    ps, ds, ls = [], [], []
    for d in range(1, min(n, 32768 + 1)):
        eq = a[d:] == a[:-d]                       # eq[j]: a[j + d] == a[j]
        m = len(eq)
        idx = np.where(~eq, np.arange(m), m)       # run of equal bytes from each j: next mismatch - j
        nxt = np.minimum.accumulate(idx[::-1])[::-1]
        run = nxt - np.arange(m)
        p = np.arange(d, n)
        length = np.minimum(np.minimum(run, 258), n - p)
        keep = length >= 3
        ps.append(p[keep]); ds.append(np.full(keep.sum(), d)); ls.append(length[keep])
    p, d, length = (np.concatenate(x) if x else np.zeros(0, np.int64) for x in (ps, ds, ls))
    order = np.lexsort((d, p))
    return p[order], d[order], length[order]


def pareto_ref(n, p, d, length):
    """per position: the candidates longer than every nearer one, the K longest of them"""
    key = p.astype(np.int64) * 512 + length
    prev = np.concatenate([[-1], np.maximum.accumulate(key)[:-1]])
    on = key > prev
    lists = np.zeros((n, K), np.uint32)
    pp, dd, ll = p[on], d[on], length[on]
    for pos in np.unique(pp):
        sel = np.where(pp == pos)[0][-K:]
        lists[pos, :len(sel)] = (ll[sel].astype(np.uint32) << 16) | (dd[sel] - 1).astype(np.uint32)
    return lists


def random_costs(seed):
    rng = random.Random(seed)
    lit = [rng.randint(4, 12) for _ in range(256)]
    lsym = {s: rng.randint(3, 12) for s in range(257, 286)}
    dsym = [rng.randint(3, 9) for _ in range(30)]
    lext = lambda s: (s - 261) // 4 if 265 <= s < 285 else 0  # noqa: E731
    lenc = [0, 0, 0] + [lsym[len_sym(x)] + lext(len_sym(x)) for x in range(3, 259)]
    distc = [dsym[s] + (s // 2 - 1 if s >= 4 else 0) for s in range(30)]
    return lit, lenc, distc


def brute_force(data, lists, lit, lenc, distc):
    n = len(data)
    best = [0] + [None] * n
    for i in range(n):
        c = best[i]
        if best[i + 1] is None or c + lit[data[i]] < best[i + 1]:
            best[i + 1] = c + lit[data[i]]
        prev = 2
        for e in lists[i]:
            if not e:
                break
            ln, d = int(e) >> 16, (int(e) & 0xFFFF) + 1
            dc = distc[dist_sym(d)]
            for x in range(prev + 1, ln + 1):
                v = c + lenc[x] + dc
                if best[i + x] is None or v < best[i + x]:
                    best[i + x] = v
            prev = ln
    return best[n]


def run_parse(emu, data, lists, costs):
    lit, lenc, distc = (np.asarray(x, np.uint32) for x in costs)
    toks = np.zeros(max(len(data), 1), np.uint32)
    cost = ctypes.c_uint64()
    nt = emu.lb2emu_parse(data, len(data), lists.ctypes.data, lit.ctypes.data, lenc.ctypes.data, distc.ctypes.data,
                          toks.ctypes.data, ctypes.byref(cost))
    return toks[:nt].tolist(), cost.value


def rebuild_and_price(tokens, costs):
    lit, lenc, distc = costs
    out, bits = bytearray(), 0
    for t in tokens:
        if t & 0x80000000:
            ln, d = ((t >> 16) & 0xFF) + 3, (t & 0x7FFF) + 1
            assert 1 <= d <= len(out)
            for _ in range(ln):
                out.append(out[-d])
            bits += lenc[ln] + distc[dist_sym(d)]
        else:
            assert t < 256
            out.append(t)
            bits += lit[t]
    return bytes(out), bits


def _text(n, seed):
    rng = random.Random(seed)
    words = [bytes(rng.choices(b"abcdefghijklmnopqrstuvwxyz", k=rng.randint(2, 9))) for _ in range(120)]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words) + rng.choice([b" ", b" ", b", ", b".\n"])
    return bytes(out[:n])


def _so_slice(n):
    path = os.path.join(HERE, "golden", "c_gold.in.bin")
    data = open(path, "rb").read()
    return data[len(data) // 3:len(data) // 3 + n]


INPUTS = {
    "random": lambda: np.random.default_rng(3).integers(0, 256, 2000, dtype=np.uint8).tobytes(),
    "runs": lambda: b"a" * 700 + b"b" * 300 + b"ab" * 100 + b"\0" * 600,
    "periodic": lambda: bytes((i * 37) & 0xFF for i in range(11)) * 150 + bytes(range(97)) * 9,
    "text": lambda: _text(2500, 5),
    "shared_object": lambda: _so_slice(2500),
    "small_alphabet": lambda: bytes(random.Random(9).choices(b"ACGT", k=2000)),
}


@pytest.mark.parametrize("name", sorted(INPUTS))
def test_parse_is_a_shortest_path_that_rebuilds_the_input(emu, name):
    data = INPUTS[name]()
    n = len(data)
    p, d, length = candidates(data)
    cand = ((length.astype(np.uint32) << 16) | (d - 1).astype(np.uint32)).astype(np.uint32)
    off = np.searchsorted(p, np.arange(n + 1)).astype(np.uint64)
    lists = np.zeros((n, K), np.uint32)
    emu.lb2emu_pareto(cand.ctypes.data, off.ctypes.data, n, lists.ctypes.data)
    assert np.array_equal(lists, pareto_ref(n, p, d, length))
    for seed in (1, 2):
        costs = random_costs(seed)
        tokens, cost = run_parse(emu, data, lists, costs)
        out, bits = rebuild_and_price(tokens, costs)
        assert out == data
        assert bits == cost == brute_force(data, lists, *costs)
        assert run_parse(emu, data, lists, costs) == (tokens, cost)


def test_equal_costs_keep_the_earliest_edge(emu):
    """With every literal and every match priced alike, many paths tie; the parse is still one fixed path: of equal
    costs, the edge that leaves the earliest position wins."""
    data = b"xyz" * 300
    n = len(data)
    p, d, length = candidates(data)
    lists = pareto_ref(n, p, d, length)
    costs = ([9] * 256, [0, 0, 0] + [9] * 256, [0] * 30)
    tokens, cost = run_parse(emu, data, lists, costs)
    assert rebuild_and_price(tokens, costs) == (data, cost)
    assert cost == brute_force(data, lists, *costs) == 9 * (3 + 4)   # xyz, then 258 * 3 + 123 = 897 in 4 matches
    assert all(run_parse(emu, data, lists, costs)[0] == tokens for _ in range(3))


def test_empty_and_tiny(emu):
    for data in (b"", b"a", b"ab", b"aaa", b"aaaa"):
        n = len(data)
        p, d, length = candidates(data)
        lists = pareto_ref(n, p, d, length) if n else np.zeros((1, K), np.uint32)
        costs = random_costs(7)
        tokens, cost = run_parse(emu, data, lists, costs)
        out, bits = rebuild_and_price(tokens, costs)
        assert out == data and bits == cost
