"""CPU checks of the dynamic-section parse behind lb2_elf_deps without a GPU: the product's parse
(lambdipy_b200/csrc/elf_deps.cuh) is compiled with g++ into a harness (tests/emu/deps_emu.cpp) that stands one thread
in for the kernels' warp, with the same count pass, scan and write pass.

* Records: on the golden inputs, every elf_fixtures variant, libraries linked with RPATH, RUNPATH, a version script
  and gold, and numpy's and scipy's shared objects, the records equal what `readelf -dVW` prints.
* Bounds: a second build under -fsanitize=address,undefined parses seeded mutants, strings cut at EOF and every
  truncation of a small object, each in a buffer of exactly its size, and must report nothing.  Where a mutant's
  parse succeeds its strings are the ones readelf reads through the same PT_DYNAMIC and DT_STRTAB (its section
  headers hidden, so that readelf cannot read the copies there instead); where readelf cannot read a string of the
  dynamic array, the parse says malformed."""
import os
import re
import struct
import subprocess

import pytest

import deps_lib as D
import elf_mutants as M
from lambdipy_b200 import _native as N


@pytest.fixture(scope="module")
def emu():
    return D.Emu()


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    return D.corpus(str(tmp_path_factory.mktemp("deps_corpus")))


def test_records_equal_readelf(emu, corpus):
    labels = sorted(corpus)
    blobs = []
    for k in labels:
        with open(corpus[k], "rb") as f:
            blobs.append(f.read())
    got = emu.parse(blobs)
    assert any(k.startswith("site/numpy") for k in labels) and any(k.startswith("site/scipy.libs") for k in labels)
    assert "variant/c_rpath_soname" in labels
    for k in ("linked/libuser_runpath.so", "linked/libuser_rpath.so", "linked/libv.so", "linked/libuser_gold.so"):
        assert k in labels, k
    for k, (status, machine, recs) in zip(labels, got):
        want, complained = D.readelf(corpus[k])
        assert not complained, k
        if k == "variant/c_static":
            assert status == N.ELF_STATIC and recs == [], k
            continue
        assert status == N.ELF_OK, (k, status)
        assert machine == 62, k
        assert recs == want, k
    kinds = {r[0] for _, _, recs in got for r in recs}
    assert kinds == set(range(1, 8))  # every record kind was met


def test_linked_tags(emu, corpus):
    """RUNPATH from --enable-new-dtags, RPATH from --disable-new-dtags; the version script's VERDEFs and their use"""
    def recs(label):
        with open(corpus[label], "rb") as f:
            return emu.parse([f.read()])[0][2]
    rt, rp = recs("linked/libuser_runpath.so"), recs("linked/libuser_rpath.so")
    assert (N.ELF_REC_RUNPATH, 0, 0, "$ORIGIN:/opt/lib") in rt and not any(r[0] == N.ELF_REC_RPATH for r in rt)
    assert (N.ELF_REC_RPATH, 0, 0, "$ORIGIN:/opt/lib") in rp and not any(r[0] == N.ELF_REC_RUNPATH for r in rp)
    assert [r[3] for r in rt if r[0] == N.ELF_REC_NEEDED][:2] == ["libv.so", "liba.so.1"]  # the link order
    v = recs("linked/libv.so")
    assert [(r[1], r[3]) for r in v if r[0] == N.ELF_REC_VERDEF] == [(1, "libv.so"), (0, "V1"), (0, "V2")]
    files = {i: r[3] for i, r in enumerate(rt) if r[0] == N.ELF_REC_VERNEED_FILE}
    assert {(files[r[2]], r[3]) for r in rt if r[0] == N.ELF_REC_VERNEED_VERSION} >= {("libv.so", "V1"), ("libv.so", "V2")}


def _asan_statuses(exe, paths):
    r = subprocess.run([exe] + paths, capture_output=True, text=True)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-4000:]
    return [int(line.split()[0]) for line in r.stdout.splitlines()]


def _no_sections(b):
    """b with e_shoff / e_shentsize / e_shnum / e_shstrndx zeroed: readelf then reads PT_DYNAMIC and DT_STRTAB"""
    m = bytearray(b)
    if len(m) >= 64:
        struct.pack_into("<Q", m, 40, 0)
        struct.pack_into("<HHH", m, 58, 0, 0, 0)
    return bytes(m)


_RAW = re.compile(r"^\s*0x[0-9a-f]+ \((NEEDED|SONAME|RPATH|RUNPATH)\)\s+0x")


def _readelf_strings(path):
    """(string records of `readelf -dW`, whether it printed a string tag as a bare number: a string it cannot read)"""
    r = subprocess.run(["readelf", "-dW", path], capture_output=True)
    out = r.stdout.decode("utf-8", "surrogateescape")
    raw = any(_RAW.match(line) for line in out.splitlines())
    return [x for x in D.readelf(path)[0] if x[0] <= N.ELF_REC_RUNPATH], raw


BASES = ("variant/c_rpath_soname", "linked/libuser_rpath.so", "linked/libuser_runpath.so", "linked/libv.so",
         "linked/libuser_gold.so", "golden/real_libXau.in.bin")


def test_mutants_under_sanitizers(emu, corpus, tmp_path):
    exe = D.asan_exe(str(tmp_path))
    bases = [corpus[k] for k in BASES]
    bases += [corpus[k] for k in sorted(corpus) if k.startswith("site/scipy.libs/libquadmath")][:1]
    seen = set()
    for bi, base in enumerate(bases):
        with open(base, "rb") as f:
            data = f.read()
        ms = list(M.mutants(data, bi))
        paths = []
        for i, (_, m) in enumerate(ms):
            p = str(tmp_path / ("m%d_%d.so" % (bi, i)))
            with open(p, "wb") as f:
                f.write(m)
            paths.append(p)
        statuses = _asan_statuses(exe, paths)
        got = emu.parse([m for _, m in ms])
        assert statuses == [g[0] for g in got]
        seen.update(statuses)
        for (label, m), (status, _, recs) in zip(ms, got):
            if label.startswith(("chain", "vna_")):
                continue  # the version chains: readelf reads them through the section headers only
            p = str(tmp_path / "view.so")
            with open(p, "wb") as f:
                f.write(_no_sections(m))
            strings, raw = _readelf_strings(p)
            if raw:
                assert status == N.ELF_MALFORMED, (base, label)
            elif status == N.ELF_OK:
                assert [r for r in recs if r[0] <= N.ELF_REC_RUNPATH] == strings, (base, label)
    assert {N.ELF_OK, N.ELF_MALFORMED, N.ELF_STATIC, N.ELF_UNSUPPORTED} <= seen


def test_version_chain_mutants(emu, corpus):
    """cyclic and oversized version chains end, malformed"""
    with open(corpus["linked/libuser_rpath.so"], "rb") as f:
        data = f.read()
    base = emu.parse([data])[0]
    assert base[0] == N.ELF_OK
    ms = [(label, m) for label, m in M.mutants(data, 0) if label.startswith(("chain", "vna_next=0", "d_val[6ffffff"))]
    got = emu.parse([m for _, m in ms])
    loops = [g[0] for (label, _), g in zip(ms, got) if label.startswith("d_val[6fffffff]=") and "=100000000" in label]
    assert loops and all(s == N.ELF_MALFORMED for s in loops)  # 2^32 Verneeds: the chain's next link 0 ends it
    assert any(g[0] == N.ELF_MALFORMED for g in got) and any(g[0] == N.ELF_OK for g in got)


def test_strings_cut_and_every_truncation(emu, corpus, tmp_path):
    exe = D.asan_exe(str(tmp_path))
    with open(corpus["variant/c_rpath_soname"], "rb") as f:
        data = f.read()
    cuts = list(range(len(data) + 1))
    blobs = [data[:k] for k in cuts]
    got = emu.parse(blobs)
    # the sanitizer build over every length, in batches of files
    step = 512
    for lo in range(0, len(cuts), step):
        paths = []
        for k in cuts[lo:lo + step]:
            p = str(tmp_path / ("t%d.so" % k))
            with open(p, "wb") as f:
                f.write(blobs[k])
            paths.append(p)
        assert _asan_statuses(exe, paths) == [g[0] for g in got[lo:lo + step]]
        for p in paths:
            os.unlink(p)
    assert got[0][0] == N.ELF_NOT_ELF and got[3][0] == N.ELF_NOT_ELF and got[10][0] == N.ELF_MALFORMED
    assert got[-1][0] == N.ELF_OK
    # a cut that leaves the dynamic array and its strings whole parses to the whole object's records
    full = got[-1][2]
    assert all(g[0] in (N.ELF_OK, N.ELF_MALFORMED, N.ELF_STATIC) for g in got[64:])
    assert all(g[2] == full for g in got if g[0] == N.ELF_OK)
