"""Package tarballs with the DEFLATE body compressed on the GPU.

The reference writes a built package with `tarfile.open(path, "w:gz")`, i.e. zlib level 9 on one core
(PackageBuild.create_compressed_tarball, lambdipy/package_build.py:165-172 of the reference).  Here the
tar stream is still written by the standard library's `tarfile`, so it is the reference's byte for byte;
only the gzip layer underneath is replaced by `GpuGzipFile`, whose DEFLATE body comes from the CUDA
encoder behind `lb2_gzip_*` (csrc/deflate.cu).  The result is an ordinary gzip file that `gzip -d`,
`tar -xzf` and `tarfile.open(..., "r:gz")` read.

    gzip_tarball(src_paths, tarball_path)          tar + gzip a list of paths, each under its basename
    create_compressed_tarball(package_build)       the reference method's mirror (patch.apply() installs it
                                                   when LAMBDIPY_TARBALL_BACKEND=b200)

Reading goes the other way: `gunzip` decodes each gzip member's DEFLATE body with the CUDA decoder behind
`lb2_inflate_*` (csrc/inflate.cu), and the standard library's `tarfile` parses and writes the tar stream.

    gunzip(path)                                   the decompressed bytes of a gzip file
    extract_tarball(tarball_path, directory)       tarfile.open(..., "r:gz").extractall(directory), inflated on the GPU
    prepare_tarfile(url, download_filename, package_directory)
                                                   the reference function's mirror (patch.apply() installs it
                                                   when LAMBDIPY_UNTAR_BACKEND=b200)
"""
import ctypes as C
import glob
import gzip
import io
import os
import struct
import tarfile
import time
import urllib.request

import numpy as np

from . import _native as N

PIECE_BYTES = 64 << 20  # input per GPU submission; two pieces are in flight while the next one is filled


class GpuGzipFile(io.BufferedIOBase):
    """Write-only gzip file whose DEFLATE body is produced on the GPU.

    The header is the one `gzip.GzipFile(path, "wb", compresslevel=9, mtime=mtime)` writes (FNAME = the
    basename without ".gz", XFL = 2, OS = 255); close() writes the CRC32 / ISIZE trailer.  `tell()` counts
    uncompressed bytes, as GzipFile's does (tarfile reads it when it opens the archive).

    ctx=None: the context the strip path has already warmed up in this process (project_build.warmup), if
    any, else a new one on device LAMBDIPY_B200_DEVICE (default 0) that close() releases.

    compresslevel=None keeps the default encoder; 9 selects the thorough one (LB2_DEFLATE_BEST: an optimal parse,
    never larger, slower); anything else raises ValueError."""

    def __init__(self, filename, mtime=None, ctx=None, piece_bytes=PIECE_BYTES, compresslevel=None):
        self.name = filename
        self._own_ctx = False
        self._ctx = self._g = self._out = self._file = None
        self._bufs = []
        flags = N.deflate_flags(compresslevel)  # checked before anything is allocated
        if ctx is None:
            ctx, self._own_ctx = _default_context()
        self._ctx = ctx
        try:
            g = C.c_void_p()
            self._ctx.check(self._ctx.lib.lb2_gzip_create(self._ctx.h, flags, C.byref(g)))
            self._g = g
            self._piece = int(piece_bytes)
            for _ in range(2):
                p = self._ctx.pinned_alloc(self._piece)
                self._bufs.append((p, np.frombuffer((C.c_uint8 * self._piece).from_address(p), dtype=np.uint8)))
            self._out_cap = N.gzip_bound(self._piece)
            self._out = self._ctx.pinned_alloc(self._out_cap)
            self._file = open(filename, "wb")
            self._file.write(gzip_header(filename, mtime))
        except BaseException:
            self._release()
            raise
        self._cur = 0          # buffer being filled
        self._fill = 0         # bytes in it
        self._in_flight = 0
        self.offset = 0        # uncompressed bytes written
        self.stats = None

    def writable(self):
        return True

    def tell(self):
        return self.offset

    def write(self, data):
        if self.closed:
            raise ValueError("write to closed file")
        src = np.frombuffer(data, dtype=np.uint8)
        n = len(src)
        pos = 0
        while pos < n:
            k = min(n - pos, self._piece - self._fill)
            self._bufs[self._cur][1][self._fill:self._fill + k] = src[pos:pos + k]
            self._fill += k
            pos += k
            if self._fill == self._piece:
                self._submit()
        self.offset += n
        return n

    def _submit(self):
        ctx = self._ctx
        ctx.check(ctx.lib.lb2_gzip_submit(self._g, self._bufs[self._cur][0], self._fill))
        self._in_flight += 1
        self._cur ^= 1
        self._fill = 0
        if self._in_flight == 2:  # the buffer to fill next belongs to the older piece: wait for it
            self._collect()

    def _collect(self):
        ctx = self._ctx
        n = C.c_uint64()
        ctx.check(ctx.lib.lb2_gzip_collect(self._g, self._out, self._out_cap, C.byref(n)))
        self._file.write(C.string_at(self._out, n.value))
        self._in_flight -= 1

    def close(self):
        if self.closed:
            return
        try:
            if self._file is not None and self._g is not None:
                if self._fill:
                    self._submit()
                while self._in_flight:
                    self._collect()
                ctx = self._ctx
                n, crc, isize, st = C.c_uint64(), C.c_uint32(), C.c_uint64(), N.GzipStats()
                ctx.check(ctx.lib.lb2_gzip_finish(self._g, self._out, self._out_cap, C.byref(n), C.byref(crc),
                                                  C.byref(isize), C.byref(st)))
                self._file.write(C.string_at(self._out, n.value))
                self._file.write(struct.pack("<II", crc.value, isize.value & 0xFFFFFFFF))
                self.stats = st.as_dict()
        finally:
            self._release()
            super().close()

    def _release(self):
        if self._file is not None:
            self._file.close()
            self._file = None
        if self._g is not None:
            self._ctx.lib.lb2_gzip_destroy(self._g)
            self._g = None
        for p, _ in self._bufs:
            self._ctx.pinned_free(p)
        self._bufs = []
        if self._out is not None:
            self._ctx.pinned_free(self._out)
            self._out = None
        if self._own_ctx and self._ctx is not None:
            self._ctx.close()
        self._ctx = None


def _default_context():
    """(context, owned by the caller)"""
    from . import project_build
    if project_build._warm is not None:
        return project_build._warm.result(), False
    return N.Context(int(os.environ.get("LAMBDIPY_B200_DEVICE", "0"))), True


def gzip_header(filename, mtime=None):
    """The 10-byte gzip header + FNAME field that gzip.GzipFile writes at compresslevel 9."""
    try:
        fname = os.path.basename(filename)
        if not isinstance(fname, bytes):
            fname = fname.encode("latin-1")
        if fname.endswith(b".gz"):
            fname = fname[:-3]
    except UnicodeEncodeError:
        fname = b""
    if mtime is None:
        mtime = time.time()
    head = struct.pack("<BBBBIBB", 0x1F, 0x8B, 8, 0x08 if fname else 0, int(mtime) & 0xFFFFFFFF, 2, 255)
    return head + (fname + b"\0" if fname else b"")


def gzip_tarball(src_paths, tarball_path, ctx=None, compresslevel=None):
    """Write `tarball_path` as a gzip-compressed tar of `src_paths`, each added recursively under its
    basename -- what `tarfile.open(tarball_path, "w:gz")` with `tar.add(p, arcname=basename(p))` writes,
    with the same tar stream.  compresslevel: as GpuGzipFile's.  Returns tarball_path."""
    N.deflate_flags(compresslevel)
    with GpuGzipFile(tarball_path, ctx=ctx, compresslevel=compresslevel) as gz, tarfile.open(name=tarball_path, mode="w", fileobj=gz) as tar:
        for path in src_paths:
            tar.add(path, arcname=os.path.basename(path))
    return tarball_path


def create_compressed_tarball(package_build, ctx=None, compresslevel=None):
    """Mirror of PackageBuild.create_compressed_tarball: every top-level entry of the package's build
    directory into ~/.lambdipy/build/<git tag>.tar.gz; returns that path.  compresslevel: as GpuGzipFile's."""
    N.deflate_flags(compresslevel)
    home = os.environ["HOME"]
    tarball_path = f"{home}/.lambdipy/build/{package_build.git_tag()}.tar.gz"
    srcs = glob.glob(f"{package_build.build_directory()}/*")
    if compresslevel is None:
        return gzip_tarball(srcs, tarball_path, ctx)
    return gzip_tarball(srcs, tarball_path, ctx, compresslevel=compresslevel)


def tarball_method(compresslevel):
    """The PackageBuild.create_compressed_tarball that patch.apply() installs: the mirror itself for the default
    encoder, else the mirror writing at `compresslevel`."""
    N.deflate_flags(compresslevel)
    if compresslevel is None:
        return create_compressed_tarball

    def create_compressed_tarball_at_level(package_build):
        return create_compressed_tarball(package_build, compresslevel=compresslevel)
    return create_compressed_tarball_at_level


# ---- reading ------------------------------------------------------------------------------------------------------
FTEXT, FHCRC, FEXTRA, FNAME, FCOMMENT = 1, 2, 4, 8, 16


class InflateDataError(gzip.BadGzipFile):
    """The DEFLATE body of a member is invalid or truncated (LB2_E_DATA)."""


def gzip_members(buf):
    """Yields the offset of each gzip member's DEFLATE body in `buf`, and expects the generator to be sent the
    number of body bytes the member used; checks framing as gzip.GzipFile does (magic, CM = 8, the FEXTRA / FNAME /
    FCOMMENT / FHCRC fields, zero padding between and after members) and refuses reserved flag bits."""
    n, pos = len(buf), 0
    while True:
        while pos < n and buf[pos] == 0:
            pos += 1
        if pos >= n:
            return
        if n - pos < 2 or bytes(buf[pos:pos + 2]) != b"\037\213":
            raise gzip.BadGzipFile("Not a gzipped file (%r)" % bytes(buf[pos:pos + 2]))
        if n - pos < 10:
            raise EOFError("Compressed file ended before the end-of-stream marker was reached")
        method, flag = buf[pos + 2], buf[pos + 3]
        if method != 8:
            raise gzip.BadGzipFile("Unknown compression method")
        if flag & 0xE0:
            raise gzip.BadGzipFile("Reserved gzip header flags set (0x%02x)" % flag)
        p = pos + 10
        if flag & FEXTRA:
            if n - p < 2:
                raise EOFError("Compressed file ended before the end-of-stream marker was reached")
            p += 2 + (buf[p] | buf[p + 1] << 8)
        for f in (FNAME, FCOMMENT):
            if flag & f:
                z = bytes(buf[p:]).find(b"\0") if p < n else -1
                if z < 0:
                    raise EOFError("Compressed file ended before the end-of-stream marker was reached")
                p += z + 1
        if flag & FHCRC:
            p += 2
        if p > n:
            raise EOFError("Compressed file ended before the end-of-stream marker was reached")
        used = yield p
        pos = p + used + 8
        if pos > n:
            raise EOFError("Compressed file ended before the end-of-stream marker was reached")


def gunzip(path, ctx=None):
    """The decompressed contents of the gzip file at `path` (all members), decoded on the GPU.

    Raises gzip.BadGzipFile for bad framing or a CRC / ISIZE mismatch, InflateDataError (a BadGzipFile) for an
    invalid DEFLATE body, EOFError for a truncated file, and NativeError with code LB2_E_CAPACITY when a member does
    not fit in device memory.  ctx=None: the context of _default_context()."""
    own = False
    if ctx is None:
        ctx, own = _default_context()
    lib, h_in, d, outs = ctx.lib, None, None, []
    try:
        size = os.path.getsize(path)
        h_in = ctx.pinned_alloc(max(size, 1))
        buf = (C.c_uint8 * size).from_address(h_in) if size else bytearray()
        with open(path, "rb") as f:
            if size and f.readinto(memoryview(buf).cast("B")) != size:
                raise EOFError("%s changed while it was read" % path)
        h = C.c_void_p()
        ctx.check(lib.lb2_inflate_create(ctx.h, 0, C.byref(h)))
        d = h
        members = gzip_members(memoryview(buf).cast("B") if size else buf)
        body = next(members, None)
        while body is not None:
            out_n, st = C.c_uint64(), N.InflateStats()
            rc = lib.lb2_inflate_run(d, h_in + body, size - body, C.byref(out_n), C.byref(st))
            if rc == N.LB2_E_DATA:
                raise InflateDataError("%s: %s" % (path, (lib.lb2_last_error(ctx.h) or b"").decode()))
            ctx.check(rc)
            crc, isize = st.crc32, out_n.value
            out = ctx.pinned_alloc(max(isize, 1))
            outs.append((out, isize))
            ctx.check(lib.lb2_inflate_read(d, out, isize))
            t = body + st.in_bytes
            if size - t < 8:
                raise EOFError("Compressed file ended before the end-of-stream marker was reached")
            want_crc, want_isize = struct.unpack_from("<II", buf, t)
            if want_crc != crc:
                raise gzip.BadGzipFile("CRC check failed")
            if want_isize != isize & 0xFFFFFFFF:
                raise gzip.BadGzipFile("Incorrect length of data produced")
            try:
                body = members.send(st.in_bytes)
            except StopIteration:
                body = None
        # the one host copy: pinned staging -> the returned bytes
        return b"".join(memoryview((C.c_uint8 * n).from_address(p)).cast("B") for p, n in outs if n)
    finally:
        if d is not None:
            lib.lb2_inflate_destroy(d)
        for p, _ in outs:
            ctx.pinned_free(p)
        if h_in is not None:
            ctx.pinned_free(h_in)
        if own:
            ctx.close()


def extract_tarball(tarball_path, directory, ctx=None):
    """tarfile.open(tarball_path, "r:gz").extractall(directory), with the gzip layer decoded on the GPU: the
    standard library still parses the tar stream and writes the files, with the running Python's defaults."""
    with tarfile.open(fileobj=io.BytesIO(gunzip(tarball_path, ctx)), mode="r:") as tar:
        tar.extractall(directory)


def prepare_tarfile(url, download_filename, package_directory):
    """Mirror of the reference's prepare_tarfile (lambdipy/project_build.py:98-102): download, then extract.  A file
    the GPU reader refuses (bad framing or data, a trailer mismatch, too large for the device) is handed to the
    reference's own two lines, which raise what the reference raises and leave what it leaves."""
    urllib.request.urlretrieve(url, download_filename)
    try:
        extract_tarball(download_filename, package_directory)
    except (gzip.BadGzipFile, EOFError) as e:
        _reference_extract(download_filename, package_directory, e)
    except N.NativeError as e:
        if e.code != N.LB2_E_CAPACITY:
            raise
        _reference_extract(download_filename, package_directory, e)


def _reference_extract(download_filename, package_directory, why):
    print("lambdipy_b200: %s: %s; extracting with tarfile" % (download_filename, why))
    tar = tarfile.open(download_filename, "r:gz")
    tar.extractall(package_directory)
    tar.close()
