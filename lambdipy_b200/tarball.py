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
"""
import ctypes as C
import glob
import io
import os
import struct
import tarfile
import time

import numpy as np

from . import _native as N

PIECE_BYTES = 64 << 20  # input per GPU submission; two pieces are in flight while the next one is filled


class GpuGzipFile(io.BufferedIOBase):
    """Write-only gzip file whose DEFLATE body is produced on the GPU.

    The header is the one `gzip.GzipFile(path, "wb", compresslevel=9, mtime=mtime)` writes (FNAME = the
    basename without ".gz", XFL = 2, OS = 255); close() writes the CRC32 / ISIZE trailer.  `tell()` counts
    uncompressed bytes, as GzipFile's does (tarfile reads it when it opens the archive).

    ctx=None: the context the strip path has already warmed up in this process (project_build.warmup), if
    any, else a new one on device LAMBDIPY_B200_DEVICE (default 0) that close() releases."""

    def __init__(self, filename, mtime=None, ctx=None, piece_bytes=PIECE_BYTES):
        self.name = filename
        self._own_ctx = False
        if ctx is None:
            ctx, self._own_ctx = _default_context()
        self._ctx = ctx
        self._g = None
        self._bufs = []
        self._out = None
        self._file = None
        try:
            g = C.c_void_p()
            self._ctx.check(self._ctx.lib.lb2_gzip_create(self._ctx.h, 0, C.byref(g)))
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


def gzip_tarball(src_paths, tarball_path, ctx=None):
    """Write `tarball_path` as a gzip-compressed tar of `src_paths`, each added recursively under its
    basename -- what `tarfile.open(tarball_path, "w:gz")` with `tar.add(p, arcname=basename(p))` writes,
    with the same tar stream.  Returns tarball_path."""
    with GpuGzipFile(tarball_path, ctx=ctx) as gz, tarfile.open(name=tarball_path, mode="w", fileobj=gz) as tar:
        for path in src_paths:
            tar.add(path, arcname=os.path.basename(path))
    return tarball_path


def create_compressed_tarball(package_build, ctx=None):
    """Mirror of PackageBuild.create_compressed_tarball: every top-level entry of the package's build
    directory into ~/.lambdipy/build/<git tag>.tar.gz; returns that path."""
    home = os.environ["HOME"]
    tarball_path = f"{home}/.lambdipy/build/{package_build.git_tag()}.tar.gz"
    return gzip_tarball(glob.glob(f"{package_build.build_directory()}/*"), tarball_path, ctx)
