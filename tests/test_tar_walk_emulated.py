"""CPU checks of the tar walk behind lb2_tar_index without a GPU: the product's walk (lambdipy_b200/csrc/tar_walk.cuh)
is compiled with g++ into a harness (tests/emu/tar_emu.cpp) that stands one thread in for the kernel's warp.

On every archive, the ranges it gathers must cover every read `tarfile.getmembers()` makes over a recording file
object, hold the archive's own bytes, and its stop offset must be where tarfile stops listing."""
import ctypes
import io
import os
import subprocess
import tarfile

import pytest

import tar_archives as A

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "tar_emu.cpp")
LIB = os.path.join(HERE, "emu", "_build_tar_emu.so")
DEPS = [SRC, os.path.join(ROOT, "lambdipy_b200", "csrc", "tar_walk.cuh")]
STOP_ZERO, STOP_BAD_HEADER, STOP_END, STOP_UNSUPPORTED = 1, 2, 3, 4


class TarEmu:
    def __init__(self):
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
            subprocess.run(["g++", "-std=c++17", "-O2", "-g", "-shared", "-fPIC", "-Wall", "-o", LIB, SRC], check=True)
        lib = self.lib = ctypes.CDLL(LIB)
        u64p, vp = ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p
        lib.lb2emu_tar_walk.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.POINTER(vp), u64p, ctypes.POINTER(vp),
                                        u64p, u64p]
        lib.lb2emu_tar_walk.restype = ctypes.c_int
        lib.lb2emu_free.argtypes = [vp]

    def walk(self, tar):
        """-> ([(off, len)], bytes, (members, stop offset, stop reason))"""
        r, b, nr, nb, res = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_uint64(), ctypes.c_uint64(), (ctypes.c_uint64 * 3)()
        assert self.lib.lb2emu_tar_walk(tar, len(tar), ctypes.byref(r), ctypes.byref(nr), ctypes.byref(b),
                                        ctypes.byref(nb), res) == 0
        flat = list((ctypes.c_uint64 * (2 * nr.value)).from_address(r.value)) if nr.value else []
        data = ctypes.string_at(b.value, nb.value) if nb.value else b""
        self.lib.lb2emu_free(r)
        self.lib.lb2emu_free(b)
        return list(zip(flat[::2], flat[1::2])), data, tuple(res)


@pytest.fixture(scope="module")
def emu():
    return TarEmu()


class Recording(io.BytesIO):
    def __init__(self, data):
        super().__init__(data)
        self.reads = []

    def read(self, n=-1):
        pos = self.tell()
        out = super().read(n)
        if out:
            self.reads.append((pos, len(out)))
        return out


def tarfile_listing(tar):
    """(reads tarfile makes to list the members, where it stops or None when it raises, members or the exception)"""
    f = Recording(tar)
    try:
        with tarfile.open(fileobj=f, mode="r:") as t:
            members = t.getmembers()
            return f.reads, t.offset, members
    except (tarfile.TarError, EOFError, IndexError) as e:
        return f.reads, None, e


def check(emu, tar, want_reason=None):
    ranges, data, (members, stop, reason) = emu.walk(tar)
    reads, t_stop, listed = tarfile_listing(tar)
    # sorted, not touching, bytes equal to the archive's
    at = 0
    for i, (off, n) in enumerate(ranges):
        assert n > 0 and (i == 0 or off > ranges[i - 1][0] + ranges[i - 1][1])
        assert data[at:at + n] == tar[off:off + n]
        at += n
    assert at == len(data)
    for pos, n in reads:
        assert any(off <= pos and pos + n <= off + ln for off, ln in ranges), (pos, n, ranges[:8])
    if t_stop is not None:
        assert stop == t_stop and members == len(listed)
    if want_reason is not None:
        assert reason == want_reason
    return ranges, reason


FORMATS = {"gnu": tarfile.GNU_FORMAT, "pax": tarfile.PAX_FORMAT, "ustar": tarfile.USTAR_FORMAT}


@pytest.mark.parametrize("fmt", sorted(FORMATS))
def test_tarfile_formats(emu, tmp_path, fmt):
    root = A.sample_tree(str(tmp_path / "pkg"))
    try:
        tar = A.tarfile_bytes(root, FORMATS[fmt])
    except ValueError:          # ustar cannot hold the long names
        tar = A.tarfile_bytes(os.path.join(root, "pkg", "lib"), FORMATS[fmt])
    check(emu, tar, STOP_ZERO)


@pytest.mark.parametrize("fmt", ["gnu", "posix", "ustar", "v7"])
def test_gnu_tar_formats(emu, tmp_path, fmt):
    root = A.sample_tree(str(tmp_path / "pkg"))
    tar = A.gnu_tar_bytes(root, fmt, str(tmp_path))
    if tar is None:             # ustar / v7 refuse the long and non-ASCII names: take the part they hold
        tar = A.gnu_tar_bytes(os.path.join(root, "pkg", "lib"), fmt, str(tmp_path))
    if tar is None:
        pytest.skip("GNU tar is not installed")
    check(emu, tar, STOP_ZERO)


@pytest.mark.parametrize("fmt", ["gnu", "posix"])
def test_gnu_sparse(emu, tmp_path, fmt):
    root = tmp_path / "sp"
    root.mkdir()
    with open(root / "holes.so", "wb") as f:
        for k in range(6):
            f.seek(k * (1 << 20))
            f.write(b"\x7fELF data %d" % k * 50)
        f.truncate(7 << 20)
    (root / "after.txt").write_bytes(b"after the sparse member\n")
    tar = A.gnu_tar_bytes(str(root), fmt, str(tmp_path), "--sparse")
    if tar is None:
        pytest.skip("GNU tar is not installed")
    check(emu, tar, STOP_ZERO)
    assert any(m.issparse() for m in tarfile.open(fileobj=io.BytesIO(tar)).getmembers())


@pytest.mark.parametrize("name", sorted(A.crafted()))
def test_crafted(emu, name):
    tar = A.crafted()[name]
    ranges, _ = check(emu, tar, STOP_ZERO)
    if name == "dir_with_size":   # the directory's size is not skipped: the next header follows it directly
        assert ranges[0] == (0, 512 * 3 + 1) or ranges[0][1] >= 1025


def test_many_members_merge(emu):
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tar:
        for i in range(500):
            ti = tarfile.TarInfo("m/%04d.txt" % i)
            ti.size = i % 3 * 700
            tar.addfile(ti, io.BytesIO(bytes(ti.size)))
    ranges, _ = check(emu, buf.getvalue(), STOP_ZERO)
    assert len(ranges) < 500          # headers of empty members merge with their neighbours


def test_damaged(emu, tmp_path):
    good = A.tarfile_bytes(A.sample_tree(str(tmp_path / "pkg")), tarfile.GNU_FORMAT)
    reasons = {}
    for name, tar in A.damaged(good).items():
        reasons[name] = check(emu, tar)[1]
    assert reasons["trailing_garbage"] == STOP_ZERO
    assert reasons["bad_checksum"] == STOP_BAD_HEADER
    assert reasons["truncated_in_header"] == reasons["no_end_marker"] == reasons["empty"] == STOP_END


def test_unsupported_stops_early(emu):
    """a GNU long name over 1 MiB: the walk stops there, and the caller fetches what follows"""
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.GNU_FORMAT) as tar:
        tar.addfile(tarfile.TarInfo("a.txt"), io.BytesIO(b""))
        tar.addfile(tarfile.TarInfo("x" * (1 << 20) + ".so"), io.BytesIO(b""))
    ranges, data, (members, stop, reason) = emu.walk(buf.getvalue())
    assert reason == STOP_UNSUPPORTED and members == 1 and stop == 512
