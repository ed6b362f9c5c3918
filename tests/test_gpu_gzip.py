"""GPU tests of the gzip writer (lb2_gzip_*, csrc/deflate.cu) and of the tarball mirror built on it.

* round trip: zlib inflates the output to the input exactly -- empty and tiny inputs, fixed-Huffman blocks with
  literals >= 0x90 (alone, as stream tails, as the only chunk of a small tar), chunk-size edges, pieces
  split at odd offsets, matches that reach across chunk and piece boundaries, long runs, incompressible data (which
  must come out as stored blocks), real shared objects; the CRC32 / ISIZE trailer values equal zlib's;
* the same input gives the same bytes on every run;
* the mirror of PackageBuild.create_compressed_tarball writes the tar stream stdlib tarfile writes, under the same
  gzip header except MTIME, and gzip / tar accept the file;
* on the numpy + scipy tree the GPU output is no larger than zlib level 1's.
"""
import ctypes as C
import filecmp
import glob
import gzip
import os
import random
import shutil
import subprocess
import tarfile
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SITE = os.path.dirname(os.path.dirname(np.__file__))


def gzip_pieces(ctx, pieces):
    """Raw API: DEFLATE the concatenation of `pieces`, one submission each (two in flight).  Returns
    (gzip file bytes, crc32, isize, stats)."""
    from lambdipy_b200 import _native as N
    from lambdipy_b200.tarball import gzip_header
    lib = ctx.lib
    g = C.c_void_p()
    ctx.check(lib.lb2_gzip_create(ctx.h, 0, C.byref(g)))
    cap = max([N.gzip_bound(len(p)) for p in pieces] + [16])
    bufs = [ctx.pinned_alloc(max([len(p) for p in pieces] + [16])) for _ in range(2)]
    out = ctx.pinned_alloc(cap)
    body, in_flight = [], []
    n = C.c_uint64()
    try:
        for i, p in enumerate(pieces):
            if len(in_flight) == 2:
                ctx.check(lib.lb2_gzip_collect(g, out, cap, C.byref(n)))
                body.append(C.string_at(out, n.value))
                in_flight.pop(0)
            buf = bufs[i & 1]
            C.memmove(buf, p, len(p))
            ctx.check(lib.lb2_gzip_submit(g, buf, len(p)))
            in_flight.append(i)
        for _ in in_flight:
            ctx.check(lib.lb2_gzip_collect(g, out, cap, C.byref(n)))
            body.append(C.string_at(out, n.value))
        crc, isize, st = C.c_uint32(), C.c_uint64(), N.GzipStats()
        ctx.check(lib.lb2_gzip_finish(g, out, cap, C.byref(n), C.byref(crc), C.byref(isize), C.byref(st)))
        body.append(C.string_at(out, n.value))
    finally:
        lib.lb2_gzip_destroy(g)
        for b in bufs:
            ctx.pinned_free(b)
        ctx.pinned_free(out)
    data = gzip_header("t.gz", 0) + b"".join(body) + crc.value.to_bytes(4, "little") + (isize.value & 0xFFFFFFFF).to_bytes(4, "little")
    return data, crc.value, isize.value, st.as_dict()


def check_round_trip(ctx, pieces):
    whole = b"".join(pieces)
    gz, crc, isize, st = gzip_pieces(ctx, pieces)
    assert zlib.decompress(gz, wbits=31) == whole
    assert crc == zlib.crc32(whole) and isize == len(whole)
    assert st["in_bytes"] == len(whole) and st["crc32"] == crc
    return gz, st


def _rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def _text(n, seed):
    rng = random.Random(seed)
    words = [bytes(rng.choices(b"abcdefghijklmnopqrstuvwxyz", k=rng.randint(2, 9))) for _ in range(400)]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words) + (b"\n" if rng.random() < 0.1 else b" ")
    return bytes(out[:n])


@pytest.mark.parametrize("n", [0, 1, 2, 3, 65535, 65536, 65537, 3 * 65536 + 1])
def test_round_trip_sizes(gpu_ctx, n):
    check_round_trip(gpu_ctx, [_text(n, n)])


@pytest.mark.parametrize("data", [b"\xff", b"\x90", b"\x8f\x90\xff", bytes(range(236, 256))])
def test_fixed_code_high_literals(gpu_ctx, data):
    """tiny inputs are cheapest with the fixed code; literals 144..255 take its 9-bit codes"""
    gz, st = check_round_trip(gpu_ctx, [data])
    assert st["n_fixed_chunks"] == 1


def test_short_random_inputs_alone_and_as_tails(gpu_ctx):
    """every length 1..800 of random bytes, alone and behind a text piece (the tail chunk of a stream);
    the short ones go through the fixed code"""
    rng = np.random.default_rng(6)
    fixed = 0
    for n in list(range(1, 64)) + [100, 150, 200, 300, 500, 800]:
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        fixed += check_round_trip(gpu_ctx, [data])[1]["n_fixed_chunks"]
        fixed += check_round_trip(gpu_ctx, [_text(65536 + 1000, n), data])[1]["n_fixed_chunks"]
    assert fixed >= 20


def test_tar_of_one_small_random_file(gpu_ctx, tmp_path):
    """a tar holding one short random file: headers, payload and zero padding in one chunk"""
    from lambdipy_b200 import tarball
    rng = np.random.default_rng(7)
    for n in (1, 200, 500, 800):
        src = tmp_path / ("src%d" % n)
        src.mkdir()
        payload = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        (src / "blob.bin").write_bytes(payload)
        out = str(tmp_path / ("t%d.tar.gz" % n))
        tarball.gzip_tarball([str(src)], out, ctx=gpu_ctx)
        with tarfile.open(out, "r:gz") as t:
            assert t.extractfile("src%d/blob.bin" % n).read() == payload


def test_round_trip_odd_piece_splits(gpu_ctx):
    data = _text(700_001, 1)
    cuts = [0, 1, 7, 7778, 65537 + 7778, 300_003, 300_004, 700_001]
    check_round_trip(gpu_ctx, [data[a:b] for a, b in zip(cuts, cuts[1:])])


def test_empty_pieces_between(gpu_ctx):
    data = _text(200_000, 2)
    check_round_trip(gpu_ctx, [b"", data[:5], b"", data[5:], b""])


def test_matches_across_chunk_and_piece_boundaries(gpu_ctx):
    block = _rand(20 * 1024, 3)
    data = block * 60                        # 1.2 MB: every copy after the first is a 20 KB-distance match
    cuts = [0, 12345, 65536 * 3 + 17, 777_777, len(data)]
    gz, st = check_round_trip(gpu_ctx, [data[a:b] for a, b in zip(cuts, cuts[1:])])
    # the random block is paid for once; every later chunk finds it in the 32 KB history, including
    # the first chunk of each piece (history from the previous piece).  Only the first piece, 12345 random
    # bytes with nothing to match, is stored.
    assert len(gz) < 3 * len(block)
    assert st["n_stored_chunks"] == 1


def test_zeros_256mb(gpu_ctx):
    gz, st = check_round_trip(gpu_ctx, [bytes(64 << 20)] * 4)
    assert len(gz) < (256 << 20) // 300       # distance-1, length-258 runs
    assert st["n_stored_chunks"] == 0


def test_incompressible_is_stored(gpu_ctx):
    from lambdipy_b200 import _native as N
    data = _rand(5 * 65536 + 999, 4)
    gz, st = check_round_trip(gpu_ctx, [data[:100_000], data[100_000:]])
    body = len(gz) - 10 - len(b"t\0") - 8
    assert body <= N.gzip_bound(100_000) + N.gzip_bound(len(data) - 100_000) + 2
    assert st["n_stored_chunks"] == st["n_chunks"] == 6


def _shared_objects(limit_bytes):
    files = sorted(glob.glob(os.path.join(SITE, "numpy", "**", "*.so"), recursive=True))
    files += sorted(glob.glob(os.path.join(SITE, "numpy.libs", "*.so*")))
    out, total = [], 0
    for f in files:
        if total >= limit_bytes:
            break
        b = open(f, "rb").read()
        out.append(b)
        total += len(b)
    assert out, "no shared objects under %s" % SITE
    return out


def test_real_shared_objects(gpu_ctx):
    blobs = _shared_objects(48 << 20)
    gz, st = check_round_trip(gpu_ctx, blobs)     # one piece per file: many piece boundaries
    assert len(gz) < sum(map(len, blobs)) * 0.6
    assert st["n_stored_chunks"] < st["n_chunks"]


def test_deterministic(gpu_ctx):
    blobs = _shared_objects(24 << 20)
    data = b"".join(blobs)
    pieces = [data[i:i + (5 << 20) + 3] for i in range(0, len(data), (5 << 20) + 3)]
    a = gzip_pieces(gpu_ctx, pieces)[0]
    b = gzip_pieces(gpu_ctx, pieces)[0]
    assert a == b


def test_gpu_gzip_file_small_pieces(gpu_ctx, tmp_path):
    """the file object: header, pieces filled across write() calls, the trailer"""
    import io
    from lambdipy_b200.tarball import GpuGzipFile
    data = _text(3_000_000, 5)
    p = tmp_path / "x.bin.gz"
    with GpuGzipFile(str(p), mtime=99, ctx=gpu_ctx, piece_bytes=1 << 20) as f:
        for i in range(0, len(data), 77_777):
            f.write(data[i:i + 77_777])
        assert f.tell() == len(data)
    assert gzip.decompress(p.read_bytes()) == data
    ref = io.BytesIO()
    with gzip.GzipFile(filename=str(p), mode="wb", compresslevel=9, fileobj=ref, mtime=99):
        pass
    hdr_len = 10 + len(b"x.bin\0")
    assert p.read_bytes()[:hdr_len] == ref.getvalue()[:hdr_len]
    assert f.stats["in_bytes"] == len(data) and f.stats["n_chunks"] == 16 + 16 + 14


# ---------------------------------------------------------------------------------------------- tarball parity
class _PackageBuild:
    def __init__(self, build_dir, tag):
        self._dir, self._tag = build_dir, tag

    def git_tag(self):
        return self._tag

    def build_directory(self):
        return self._dir


def _fixture_tree(root):
    shutil.copytree(os.path.join(SITE, "numpy"), os.path.join(root, "numpy"), symlinks=True,
                    ignore=shutil.ignore_patterns("__pycache__"))
    os.symlink("numpy/__init__.py", os.path.join(root, "link_to_init.py"))
    os.mkdir(os.path.join(root, "empty_dir"))
    deep = os.path.join(root, "deep", "d" * 60)
    os.makedirs(deep)
    with open(os.path.join(deep, "f" * 90 + ".txt"), "w") as f:      # path > 100 bytes: PAX header
        f.write("long name\n" * 100)
    with open(os.path.join(root, "données_ünïcödé_名前.py"), "w", encoding="utf-8") as f:
        f.write("# non-ASCII name\n")


def _trees_equal(a, b):
    cmp = filecmp.dircmp(a, b)
    assert not cmp.left_only and not cmp.right_only and not cmp.diff_files and not cmp.funny_files, cmp.report()
    for name in cmp.common:
        pa, pb = os.path.join(a, name), os.path.join(b, name)
        assert os.path.islink(pa) == os.path.islink(pb)
        if os.path.islink(pa):
            assert os.readlink(pa) == os.readlink(pb)
        elif os.path.isdir(pa):
            _trees_equal(pa, pb)
        else:
            assert open(pa, "rb").read() == open(pb, "rb").read(), name


def test_tarball_parity_with_stdlib(gpu_ctx, tmp_path, monkeypatch):
    from lambdipy_b200 import tarball
    home = tmp_path / "home"
    build = home / ".lambdipy" / "build" / "numpy" / "1.0"
    build.mkdir(parents=True)
    _fixture_tree(str(build))
    monkeypatch.setenv("HOME", str(home))
    pb = _PackageBuild(str(build), "numpy-1.0-1")

    path = tarball.create_compressed_tarball(pb, ctx=gpu_ctx)
    assert path == "%s/.lambdipy/build/numpy-1.0-1.tar.gz" % home
    ref_path = str(tmp_path / "numpy-1.0-1.tar.gz")
    with tarfile.open(ref_path, "w:gz") as tar:
        for p in glob.glob(f"{pb.build_directory()}/*"):
            tar.add(p, arcname=os.path.basename(p))

    mine, ref = open(path, "rb").read(), open(ref_path, "rb").read()
    assert gzip.decompress(mine) == gzip.decompress(ref)
    name_end = 10 + len(b"numpy-1.0-1.tar\0")
    assert mine[:4] == ref[:4] and mine[8:name_end] == ref[8:name_end]    # all but MTIME
    names = tarfile.open(path, "r:gz").getnames()
    assert any(len(n) > 100 for n in names) and "empty_dir" in names and "link_to_init.py" in names

    out_a, out_b = tmp_path / "a", tmp_path / "b"
    for src, dst in ((path, out_a), (ref_path, out_b)):
        with tarfile.open(src, "r:gz") as t:
            t.extractall(dst, filter="tar")
    _trees_equal(str(out_a), str(out_b))

    if shutil.which("gzip"):
        subprocess.run(["gzip", "-t", path], check=True)
    if shutil.which("tar"):
        r = subprocess.run(["tar", "-tzf", path], check=True, capture_output=True)
        assert len(r.stdout.splitlines()) == len(names)


# ---------------------------------------------------------------------------------------------- ratio
def _numpy_scipy_tar():
    import io
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w") as tar:
        for d in ("numpy", "numpy.libs", "scipy", "scipy.libs"):
            p = os.path.join(SITE, d)
            if os.path.exists(p):
                tar.add(p, arcname=d)
    return buf.getvalue()


def test_ratio_not_worse_than_zlib_level1(gpu_ctx):
    if not os.path.isdir(os.path.join(SITE, "scipy")):
        pytest.skip("scipy is not installed")
    data = _numpy_scipy_tar()
    piece = 64 << 20
    gz, crc, isize, st = gzip_pieces(gpu_ctx, [data[i:i + piece] for i in range(0, len(data), piece)])
    assert crc == zlib.crc32(data) and isize == len(data)
    gpu = len(gz) / len(data)
    lvl1 = len(zlib.compress(data, 1)) / len(data)
    print("numpy+scipy tar: %d bytes, GPU ratio %.4f, zlib-1 %.4f" % (len(data), gpu, lvl1))
    assert gpu <= lvl1
    assert zlib.decompress(gz, wbits=31) == data
