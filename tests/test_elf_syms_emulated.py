"""CPU checks of the symbol index behind lb2_syms_* without a GPU: the product's logic (lambdipy_b200/csrc/elf_syms.cuh)
is compiled with g++ into a harness (tests/emu/syms_emu.cpp) that stands one thread in for each warp.

* each object's references are the symbols `readelf -rsW` shows relocations naming with an UND, non-LOCAL symbol, on
  the golden inputs, the elf_fixtures variants, the linked libraries and numpy's and scipy's shared objects;
* an ASan + UBSan build indexes and resolves seeded mutants of the fields the index reads (hash tables, versym,
  relocation sizes, symbol indices past the count, DT_RELAENT, version chains) and every truncation of a 16 KB
  object, reading no byte outside the buffers."""
import random
import struct
import subprocess

import pytest

import deps_lib as D
import syms_lib as S
from lambdipy_b200 import _native as N


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    return D.corpus(str(tmp_path_factory.mktemp("syms_corpus")))


def test_references_equal_readelf(corpus):
    emu = S.EmuResolver()
    labels = sorted(corpus)
    blobs = []
    for k in labels:
        with open(corpus[k], "rb") as f:
            blobs.append(f.read())
    checked = 0
    for k, (i, status, nrefs) in zip(labels, emu.index_blobs(blobs)):
        if status != N.SYM_OK:
            assert status in (N.ELF_STATIC, N.ELF_NOT_ELF), (k, status)
            continue
        got = {r[1] for r in emu.refs(i)}
        assert got == {name for name, _ in S.readelf_refs(corpus[k])}, k
        assert nrefs == len(emu.refs(i)) and len(got) == nrefs, k
        checked += 1
    assert checked > 100


def _dyn(data):
    """{tag: (file offset of the entry, value)} of the dynamic array (last entry of a tag), and the PT_LOAD mapping"""
    phoff, phnum = struct.unpack_from("<Q", data, 32)[0], struct.unpack_from("<H", data, 56)[0]
    loads, dyn = [], None
    for i in range(phnum):
        t, _, off, va, _, fs = struct.unpack_from("<IIQQQQ", data, phoff + 56 * i)
        if t == 1:
            loads.append((va, off, fs))
        elif t == 2:
            dyn = (off, fs)
    tags, o = {}, dyn[0]
    while o + 16 <= dyn[0] + dyn[1]:
        tag, val = struct.unpack_from("<qQ", data, o)
        if tag == 0:
            break
        tags[tag] = (o, val)
        o += 16
    return tags, lambda va: next(off + va - v for v, off, fs in loads if v <= va < v + fs)


DT_HASH, DT_SYMTAB, DT_RELA, DT_RELASZ, DT_RELAENT, DT_JMPREL, DT_PLTRELSZ = 4, 6, 7, 8, 9, 23, 2
DT_GNU_HASH, DT_VERSYM, DT_VERNEED, DT_VERDEF = 0x6ffffef5, 0x6ffffff0, 0x6ffffffe, 0x6ffffffc


def symbol_mutants(data, seed):
    """[(label, bytes)]: seeded edits of the fields the index reads"""
    rnd = random.Random(seed)
    tags, off_of = _dyn(data)
    out = []

    def put(label, at, fmt, value):
        b = bytearray(data)
        struct.pack_into(fmt, b, at, value)
        out.append((label, bytes(b)))
    for tag in (DT_GNU_HASH, DT_HASH):
        if tag in tags:
            h = off_of(tags[tag][1])
            for k in range(4):
                for v in (0, 1, 0xffffffff, rnd.randrange(1 << 32), 3, 64):
                    put("hash%x+%d=%d" % (tag, 4 * k, v), h + 4 * k, "<I", v)
            for k in range(20):  # buckets and chains
                put("hash%x word %d" % (tag, k), h + 16 + 4 * rnd.randrange(64), "<I", rnd.choice([0, 1, 0xffffffff, rnd.randrange(1 << 20)]))
    for tag in (DT_RELASZ, DT_PLTRELSZ, DT_RELAENT):
        if tag in tags:
            for v in (0, 8, 23, 25, 48, tags[tag][1] + 24, 1 << 40):
                put("tag%x=%d" % (tag, v), tags[tag][0] + 8, "<Q", v)
    for tag in (DT_RELA, DT_JMPREL):
        if tag in tags:
            r = off_of(tags[tag][1])
            for k in range(10):  # a symbol index past the count, or anywhere
                put("rel sym %d" % k, r + 24 * rnd.randrange(4) + 12, "<I", rnd.choice([1 << 20, 0xffffffff, rnd.randrange(64)]))
    if DT_VERSYM in tags:
        v = off_of(tags[DT_VERSYM][1])
        for k in range(10):
            put("versym %d" % k, v + 2 * rnd.randrange(64), "<H", rnd.choice([0x7fff, 0x8003, 2, 3, 0xffff]))
    for tag in (DT_VERNEED, DT_VERDEF):
        if tag in tags:
            v = off_of(tags[tag][1])
            put("ver loop %x" % tag, v + (12 if tag == DT_VERNEED else 16), "<I", 0)
            put("ver aux loop %x" % tag, v + 8 if tag == DT_VERNEED else v + 12, "<I", 0)
            put("ver ndx %x" % tag, v + 4, "<H", 0x7fff)
    for tag in (DT_SYMTAB, DT_GNU_HASH, DT_VERSYM, DT_RELA):
        if tag in tags:
            put("addr%x" % tag, tags[tag][0] + 8, "<Q", rnd.choice([1, 1 << 40, tags[tag][1] + len(data)]))
    put("syment", tags[DT_SYMTAB][0], "<q", 11)  # the DT_SYMTAB entry made DT_SYMENT 11 with its address as value
    return out


def test_asan_mutants_and_truncations(corpus, tmp_path):
    exe = S.asan_exe(str(tmp_path))
    small = D.linked_corpus(str(tmp_path / "linked"))
    bases = [corpus["golden/c_plain.in.bin"], corpus["golden/cxx_g.in.bin"], small["libv.so"], small["libuser_rpath.so"],
             small["libuser_gold.so"]]
    statuses = set()
    for bi, base in enumerate(bases):
        with open(base, "rb") as f:
            data = f.read()
        files = []
        for j, (label, m) in enumerate(symbol_mutants(data, bi)):
            p = tmp_path / ("m%d_%d" % (bi, j))
            p.write_bytes(m)
            files.append(str(p))
        r = subprocess.run([exe] + files, capture_output=True, text=True)
        assert r.returncode == 0, (base, r.stderr[-3000:])
        statuses |= {int(line.split()[0]) for line in r.stdout.splitlines()}
    assert {N.SYM_OK, N.SYM_MALFORMED} <= statuses
    # every truncation of a small object (about 16 KB)
    with open(small["libuser_rpath.so"], "rb") as f:
        data = f.read()
    assert len(data) <= 20000
    files = []
    for n in range(len(data) + 1):
        p = tmp_path / ("t%d" % n)
        p.write_bytes(data[:n])
        files.append(str(p))
    for k in range(0, len(files), 400):
        r = subprocess.run([exe] + files[k:k + 400], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
    full = subprocess.run([exe, small["libuser_rpath.so"]], capture_output=True, text=True).stdout.split()
    assert full[0] == "0" and int(full[2]) > 0


def test_dt_rel_and_bad_entry_size_are_refused(corpus):
    with open(corpus["golden/c_plain.in.bin"], "rb") as f:
        data = f.read()
    tags, _ = _dyn(data)
    emu = S.EmuResolver()
    b = bytearray(data)
    struct.pack_into("<q", b, tags[DT_RELAENT][0], 17)  # DT_RELAENT's entry retagged DT_REL
    bad = bytearray(data)
    struct.pack_into("<Q", bad, tags[DT_RELAENT][0] + 8, 16)
    got = emu.index_blobs([data, bytes(b), bytes(bad)])
    assert [g[1] for g in got] == [N.SYM_OK, N.SYM_UNSUPPORTED, N.SYM_MALFORMED]
