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

Both chained on the device: `strip_tarball` strips the shared objects inside a package tarball without unpacking it.
The tar stream is inflated into device memory, one warp walks its headers (`lb2_tar_index`, csrc/tar.cu) so that
tarfile lists the members from one download, the `*.so` members are stripped where they lie, and the new tar stream is
deflated from device segments (`lb2_gzip_submit_device`).

    strip_tarball(src, dst)                        the .tar.gz that extracting src, the reference's
                                                   `find -name "*.so" | xargs strip` and tarfile "w:gz" would give
    python -m lambdipy_b200.tarball strip SRC DST [--level 9] [--seek-table]

With seek_table=True the writers append a seek table (seek_table.py): the compressed and decoded length of every
64 KB chunk, which the encoder computes anyway.  The readers find it from the file's tail and decode each chunk once
from its known start (lb2_inflate_run_table) instead of searching for block starts; a table the reader does not
accept costs one decode pass and the file is then read by the search, with the same bytes.
"""
import ctypes as C
import glob
import gzip
import io
import os
import posixpath
import struct
import tarfile
import tempfile
import time
import urllib.request

import numpy as np

from . import _native as N
from . import seek_table as ST

PIECE_BYTES = 64 << 20  # input per GPU submission; two pieces are in flight while the next one is filled


class GpuGzipFile(io.BufferedIOBase):
    """Write-only gzip file whose DEFLATE body is produced on the GPU.

    The header is the one `gzip.GzipFile(path, "wb", compresslevel=9, mtime=mtime)` writes (FNAME = the
    basename without ".gz", XFL = 2, OS = 255); close() writes the CRC32 / ISIZE trailer.  `tell()` counts
    uncompressed bytes, as GzipFile's does (tarfile reads it when it opens the archive).

    ctx=None: the context the strip path has already warmed up in this process (project_build.warmup), if
    any, else a new one on device LAMBDIPY_B200_DEVICE (default 0) that close() releases.

    compresslevel=None keeps the default encoder; 9 selects the thorough one (LB2_DEFLATE_BEST: an optimal parse,
    never larger, slower); anything else raises ValueError.

    seek_table=True appends a seek table (seek_table.py) after the trailer when the stream has two or more entries:
    the chunk sizes the encoder already computes, with which the GPU reader decodes the file in one pass, without
    searching for block starts.  The bytes before it are the ones written without it."""

    def __init__(self, filename, mtime=None, ctx=None, piece_bytes=PIECE_BYTES, compresslevel=None, fileobj=None,
                 host_buffers=True, seek_table=False):
        self.name = filename
        self._own_ctx = False
        self._ctx = self._g = self._out = self._file = None
        self._own_file = fileobj is None
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
            for _ in range(2 if host_buffers else 0):
                p = self._ctx.pinned_alloc(self._piece)
                self._bufs.append((p, np.frombuffer((C.c_uint8 * self._piece).from_address(p), dtype=np.uint8)))
            self._out_cap = N.gzip_bound(self._piece)
            self._out = self._ctx.pinned_alloc(self._out_cap)
            self._file = open(filename, "wb") if fileobj is None else fileobj
            self._file.write(gzip_header(filename, mtime))
        except BaseException:
            self._release()
            raise
        self._cur = 0          # buffer being filled
        self._fill = 0         # bytes in it
        self._in_flight = 0
        self.offset = 0        # uncompressed bytes written
        self.stats = None
        self._seek = bool(seek_table)
        self._pending = []     # uncompressed bytes of each piece in flight, oldest first
        self._chunks = []      # (compressed, uncompressed) of every collected chunk

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
        self._pending.append(self._fill)
        self._in_flight += 1
        self._cur ^= 1
        self._fill = 0
        if self._in_flight == 2:  # the buffer to fill next belongs to the older piece: wait for it
            self._collect()

    def submit_device(self, refs):
        """Appends one piece whose bytes already lie in device memory: refs [(device address, length)], taken back to
        back (lb2_gzip_submit_device).  Pieces of exactly piece_bytes, the last one shorter, give the bytes write()
        gives for the concatenation.  The sources must stay unchanged until close() returns."""
        if self.closed:
            raise ValueError("write to closed file")
        if self._fill:
            raise ValueError("submit_device after a partial write(): the piece boundaries would differ")
        ctx = self._ctx
        src = (N.ZipSource * max(len(refs), 1))()
        for i, (addr, n) in enumerate(refs):
            src[i].d_ptr, src[i].len = addr, n
        ctx.check(ctx.lib.lb2_gzip_submit_device(self._g, src, len(refs)))
        self._pending.append(sum(n for _, n in refs))
        self._in_flight += 1
        self.offset += sum(n for _, n in refs)
        if self._in_flight == 2:  # keep one piece running while the older one is collected
            self._collect()

    def _collect(self):
        ctx = self._ctx
        n = C.c_uint64()
        ctx.check(ctx.lib.lb2_gzip_collect(self._g, self._out, self._out_cap, C.byref(n)))
        self._file.write(C.string_at(self._out, n.value))
        self._in_flight -= 1
        size = self._pending.pop(0)
        if self._seek:
            k = C.c_uint32()
            sizes = (C.c_uint32 * max(-(-size // ST.CHUNK), 1))()
            ctx.check(ctx.lib.lb2_gzip_chunk_sizes(self._g, sizes, len(sizes), C.byref(k)))
            if k.value != -(-size // ST.CHUNK) or sum(sizes[:k.value]) != n.value:
                raise RuntimeError("lb2_gzip_chunk_sizes: %d chunks of %d bytes for a piece of %d bytes in %d"
                                   % (k.value, sum(sizes[:k.value]), size, n.value))
            self._chunks += [(sizes[i], min(ST.CHUNK, size - i * ST.CHUNK)) for i in range(k.value)]

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
                if self._seek and self._chunks:
                    c, u = self._chunks[-1]
                    self._chunks[-1] = (c + n.value, u)   # the final block belongs to the last entry
                    entries = ST.build(self._chunks)
                    self.stats["seek_entries"] = len(entries) if entries else 0
                    if entries:
                        self._file.write(ST.gzip_member(entries, self._file.tell()))
        finally:
            self._release()
            super().close()

    def _release(self):
        if self._file is not None:
            if self._own_file:
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


def gzip_tarball(src_paths, tarball_path, ctx=None, compresslevel=None, seek_table=False):
    """Write `tarball_path` as a gzip-compressed tar of `src_paths`, each added recursively under its
    basename -- what `tarfile.open(tarball_path, "w:gz")` with `tar.add(p, arcname=basename(p))` writes,
    with the same tar stream.  compresslevel, seek_table: as GpuGzipFile's.  Returns tarball_path."""
    N.deflate_flags(compresslevel)
    with GpuGzipFile(tarball_path, ctx=ctx, compresslevel=compresslevel, seek_table=seek_table) as gz, \
            tarfile.open(name=tarball_path, mode="w", fileobj=gz) as tar:
        for path in src_paths:
            tar.add(path, arcname=os.path.basename(path))
    return tarball_path


def create_compressed_tarball(package_build, ctx=None, compresslevel=None, seek_table=False):
    """Mirror of PackageBuild.create_compressed_tarball: every top-level entry of the package's build
    directory into ~/.lambdipy/build/<git tag>.tar.gz; returns that path.  compresslevel, seek_table: as
    GpuGzipFile's."""
    N.deflate_flags(compresslevel)
    home = os.environ["HOME"]
    tarball_path = f"{home}/.lambdipy/build/{package_build.git_tag()}.tar.gz"
    srcs = glob.glob(f"{package_build.build_directory()}/*")
    level = {} if compresslevel is None and not seek_table else {"compresslevel": compresslevel}
    return gzip_tarball(srcs, tarball_path, ctx, **level, **ST.seek_kw(seek_table))


def tarball_method(compresslevel, seek_table=False):
    """The PackageBuild.create_compressed_tarball that patch.apply() installs: the mirror itself for the default
    encoder without a seek table, else the mirror writing at `compresslevel`, with a seek table if asked."""
    N.deflate_flags(compresslevel)
    if compresslevel is None and not seek_table:
        return create_compressed_tarball

    def create_compressed_tarball_at_level(package_build):
        return create_compressed_tarball(package_build, compresslevel=compresslevel, **ST.seek_kw(seek_table))
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
    lib, d, outs = ctx.lib, None, []
    try:
        h = C.c_void_p()
        ctx.check(lib.lb2_inflate_create(ctx.h, 0, C.byref(h)))
        d = h

        def keep(isize, last, st):
            out = ctx.pinned_alloc(max(isize, 1))
            outs.append((out, isize))
            ctx.check(lib.lb2_inflate_read(d, out, isize))
        inflate_members(ctx, d, path, keep)
        # the one host copy: pinned staging -> the returned bytes
        return b"".join(memoryview((C.c_uint8 * n).from_address(p)).cast("B") for p, n in outs if n)
    finally:
        if d is not None:
            lib.lb2_inflate_destroy(d)
        for p, _ in outs:
            ctx.pinned_free(p)
        if own:
            ctx.close()


def _seek_spans(buf, size):
    """(where the members end, the lb2_inflate_span table of the first member, or None): a file of exactly one data
    member followed by a seek-table member whose entries add up to that member's body and ISIZE.  Anything else reads
    as a file without a table (its last member, if any, is then an empty gzip member like any other)."""
    tail = ST.gzip_tail(memoryview(buf).cast("B")) if size else None
    if tail is None:
        return size, None
    end, entries = tail
    try:
        body = next(gzip_members(memoryview(buf).cast("B")[:end]), None)
    except (gzip.BadGzipFile, EOFError):
        return size, None
    if body is None or body > end - 8 or buf[0] == 0:
        return size, None
    if not ST.valid(entries, end - 8 - body, struct.unpack_from("<I", buf, end - 4)[0], 0xFFFFFFFF):
        return size, None
    spans = (N.InflateSpan * len(entries))()
    for i, (c, u) in enumerate(entries):
        spans[i].in_len, spans[i].out_len = c, u
    return end, spans


def inflate_members(ctx, d, path, on_member, counts=None):
    """Reads the gzip file at `path` into pinned memory and decodes each member's DEFLATE body with the reader `d`
    (lb2_inflate_run), checking framing, CRC-32 and ISIZE; raises what gunzip raises.  After each member,
    on_member(isize, last, stats) is called while its bytes are still the reader's output (`last`: no member follows;
    stats: its N.InflateStats).  A file written with a seek table (seek_table.py) is decoded from the table
    (lb2_inflate_run_table) and its table member is not a member here; counts (a dict, may be None) then gains
    seek_table 1, or seek_table_refused 1 when the reader did not accept the table and searched instead.
    Returns (the first member's MTIME or None, the bytes uploaded)."""
    lib, h_in, mtime, uploaded = ctx.lib, None, None, 0
    try:
        size = os.path.getsize(path)
        h_in = ctx.pinned_alloc(max(size, 1))
        buf = (C.c_uint8 * size).from_address(h_in) if size else bytearray()
        with open(path, "rb") as f:
            if size and f.readinto(memoryview(buf).cast("B")) != size:
                raise EOFError("%s changed while it was read" % path)
        end, spans = _seek_spans(buf, size)
        members = gzip_members(memoryview(buf).cast("B")[:end] if size else buf)
        body = next(members, None)
        if body is not None:
            start = next(i for i in range(size) if buf[i])
            mtime = struct.unpack_from("<I", buf, start + 4)[0]
        while body is not None:
            out_n, st = C.c_uint64(), N.InflateStats()
            if spans is not None:
                used, refused = C.c_uint32(), C.c_uint32()
                rc = lib.lb2_inflate_run_table(d, h_in + body, size - body, spans, len(spans), C.byref(out_n),
                                               C.byref(st), C.byref(used), C.byref(refused))
                if counts is not None:
                    counts["seek_table"] = counts.get("seek_table", 0) + used.value
                    counts["seek_table_refused"] = counts.get("seek_table_refused", 0) + refused.value
                spans = None
            else:
                rc = lib.lb2_inflate_run(d, h_in + body, size - body, C.byref(out_n), C.byref(st))
            uploaded += size - body
            if rc == N.LB2_E_DATA:
                raise InflateDataError("%s: %s" % (path, (lib.lb2_last_error(ctx.h) or b"").decode()))
            ctx.check(rc)
            crc, isize = st.crc32, out_n.value
            t = body + st.in_bytes
            if size - t < 8:
                raise EOFError("Compressed file ended before the end-of-stream marker was reached")
            want_crc, want_isize = struct.unpack_from("<II", buf, t)
            if want_crc != crc:
                raise gzip.BadGzipFile("CRC check failed")
            if want_isize != isize & 0xFFFFFFFF:
                raise gzip.BadGzipFile("Incorrect length of data produced")
            k = t + 8
            while k < end and buf[k] == 0:
                k += 1
            on_member(isize, k >= end, st)
            try:
                body = members.send(st.in_bytes)
            except StopIteration:
                body = None
        return mtime, uploaded
    finally:
        if h_in is not None:
            ctx.pinned_free(h_in)


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


# ---- strip_tarball: inflate, strip and deflate chained on the device ----------------------------------------------
# Four seams, each an object a CPU stand-in can replace: the reader (the tar stream decoded into one device buffer),
# the index (the bytes tarfile reads to list the members), the stripper (zipfile_gpu.GpuStripper) and the writer
# (GpuGzipFile fed from device memory).  What travels between them is a reference, a (device address, length) pair.

RECORDSIZE = tarfile.RECORDSIZE
BLOCKSIZE = tarfile.BLOCKSIZE
_SYMLINK_HOPS = 40


class GpuTarReader:
    """The tar stream of a gzip file decoded on the GPU and left in device memory.

    read(path) -> ((address, length) of the whole tar stream, the first member's MTIME): a single-member file stays in
    the reader's own output buffer (lb2_inflate_device_output), the members of a multi-member file are concatenated
    into one device arena (lb2_memcpy_d2d); either is 256-byte aligned and valid until close().  fetch(address, n)
    copies device bytes to the host, upload(data) puts bytes on the device, zeros(n) is a zeroed device buffer; all
    of them stay valid until close()."""

    def __init__(self, ctx):
        self._ctx, self._d, self._arena, self._extra = ctx, None, None, []
        self.uploaded = self.downloaded = 0
        self._stats = {}
        d = C.c_void_p()
        ctx.check(ctx.lib.lb2_inflate_create(ctx.h, 0, C.byref(d)))
        self._d = d

    def _alloc(self, n):
        try:
            return self._ctx.dev_alloc(n)
        except N.NativeError as e:
            raise N.NativeError(N.LB2_E_CAPACITY, "the tar stream does not fit in device memory (%s)" % e) from None

    def _decode(self, path, state, in_place):
        """inflate_members on `path`, every member appended to the arena at state["fill"]; in_place: a file of one
        member is left in the reader's output buffer instead and state["ref"] is set to it.  Returns the MTIME."""
        ctx, lib = self._ctx, self._ctx.lib

        def on_member(isize, last, st):
            for k, v in st.as_dict().items():
                if k.endswith("_ms") or k.startswith("n_"):
                    self._stats[k] = self._stats.get(k, 0) + v
            d_out, n = C.c_void_p(), C.c_uint64()
            ctx.check(lib.lb2_inflate_device_output(self._d, C.byref(d_out), C.byref(n)))
            if in_place and state["ref"] is None and state["fill"] == 0 and last:
                state["ref"] = (d_out.value or 0, n.value)    # the only member: used where it lies
                return
            need = state["fill"] + isize
            if need > state["cap"]:
                cap = -(-max(need, 2 * state["cap"], 1 << 20) // 256) * 256   # read_many's next start stays inside
                arena = self._alloc(cap)
                if state["fill"]:
                    ctx.d2d(arena, self._arena, state["fill"])
                if self._arena is not None:
                    ctx.dev_free(self._arena)
                self._arena, state["cap"] = arena, cap
            if isize:
                ctx.d2d(self._arena + state["fill"], d_out.value, isize)
            state["fill"] = need

        mtime, uploaded = inflate_members(ctx, self._d, path, on_member, self._stats)
        self.uploaded += uploaded
        return mtime

    def read(self, path):
        state = {"ref": None, "fill": 0, "cap": 0}
        self.uploaded = 0
        mtime = self._decode(path, state, True)
        ref = state["ref"] or ((self._arena or 0), state["fill"])
        return ref, mtime

    def read_many(self, paths):
        """The tar streams of several gzip files in one device arena, each at a 256-byte-aligned offset: [(address,
        length)] in the order of `paths`, valid until close().  One file is read() as it is."""
        if len(paths) == 1:
            return [self.read(paths[0])[0]]
        state, spans = {"ref": None, "fill": 0, "cap": 0}, []
        self.uploaded = 0
        for path in paths:
            state["fill"] = start = -(-state["fill"] // 256) * 256
            self._decode(path, state, False)
            spans.append((start, state["fill"] - start))
        return [((self._arena or 0) + off, n) for off, n in spans]   # the arena moves while it grows

    def fetch(self, addr, n):
        buf = C.create_string_buffer(n)
        if n:
            self._ctx.d2h(buf, addr, n)
        self.downloaded += n
        return buf.raw

    def upload(self, data):
        p = self._ctx.dev_alloc(max(len(data), 1))
        self._extra.append(p)
        if data:
            self._ctx.h2d(p, bytes(data), len(data))
        self.uploaded += len(data)
        return p

    def zeros(self, n):
        p = self._ctx.dev_alloc(n)
        self._extra.append(p)
        self._ctx.check(self._ctx.lib.lb2_memset_d(self._ctx.h, p, 0, n))
        return p

    def stats(self):
        d = dict(self._stats)
        d["kernel_ms"] = sum(d.get(k, 0.0) for k in ("find_ms", "count_ms", "decode_ms", "resolve_ms", "crc_ms"))
        return d

    def close(self):
        for p in self._extra:
            self._ctx.dev_free(p)
        self._extra = []
        if self._arena is not None:
            self._ctx.dev_free(self._arena)
            self._arena = None
        if self._d is not None:
            self._ctx.lib.lb2_inflate_destroy(self._d)
            self._d = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class GpuTarIndex:
    """lb2_tar_index: index((address, length)) -> ([(off, len)] ranges, their bytes back to back, stats dict)."""

    def __init__(self, ctx):
        self._ctx = ctx

    def index(self, ref):
        ctx, lib = self._ctx, self._ctx.lib
        addr, n = ref
        max_ranges, cap = min(n // BLOCKSIZE + 2, 1 << 15), min(n + 1, 8 << 20)
        while True:
            ranges, data = (N.TarRange * max(max_ranges, 1))(), C.create_string_buffer(max(cap, 1))
            nr, nb, st = C.c_uint32(), C.c_uint64(), N.TarIndexStats()
            rc = lib.lb2_tar_index(ctx.h, addr or None, n, ranges, max_ranges, C.byref(nr), data, cap, C.byref(nb),
                                   C.byref(st))
            if rc == N.LB2_E_CAPACITY and (nr.value > max_ranges or nb.value > cap):
                max_ranges, cap = nr.value, nb.value
                continue
            ctx.check(rc)
            break
        return [(ranges[i].off, ranges[i].len) for i in range(nr.value)], data.raw[:nb.value], st.as_dict()


class IndexedView:
    """A read-only file over a tar stream of n bytes in device memory, for tarfile to list the members from: a read
    inside one of the gathered ranges is served from their bytes, anything else is fetched with fetch(off, n) and
    counted as a miss."""

    def __init__(self, n, ranges, data, fetch):
        self._n, self._fetch, self._pos = n, fetch, 0
        self._starts, self._ends, self._at = [], [], []
        k = 0
        for off, ln in ranges:
            self._starts.append(off)
            self._ends.append(off + ln)
            self._at.append(k)
            k += ln
        self._data = data
        self.misses = self.miss_bytes = 0

    def tell(self):
        return self._pos

    def seek(self, off, whence=0):
        self._pos = off if whence == 0 else self._pos + off if whence == 1 else self._n + off
        return self._pos

    def read(self, size=-1):
        import bisect
        pos = self._pos
        end = self._n if size is None or size < 0 else min(self._n, pos + size)
        if pos >= end:
            return b""
        i = bisect.bisect_right(self._starts, pos) - 1
        if i >= 0 and self._ends[i] >= end:
            out = self._data[self._at[i] + pos - self._starts[i]:self._at[i] + end - self._starts[i]]
        else:
            out = self._fetch(pos, end - pos)
            self.misses += 1
            self.miss_bytes += end - pos
        self._pos = end
        return out


def list_members(ref, indexer, reader):
    """tarfile's member list of the tar stream at ref = (address, length) in device memory, read from one index
    download: (members, the offset tarfile stopped at, the IndexedView, (ranges, their bytes, the index's stats))."""
    base, n = ref
    ranges, data, ist = indexer.index(ref)
    view = IndexedView(n, ranges, data, lambda off, k: reader.fetch(base + off, k))
    with tarfile.open(fileobj=view, mode="r:") as tar:
        members = tar.getmembers()
        stop = tar.offset
    return members, stop, view, (ranges, data, ist)


def _norm(name):
    return posixpath.normpath(name) if name else name


def _leaves(path):
    return path.startswith("/") or path == ".." or path.startswith("../")


def _resolve(path, final, hops):
    """The member a path of the extracted tree ends at: every component that is a symlink member (the last member of
    that name) is replaced by its target, relative to the link's directory; None when it dangles, leaves the archive
    or takes more than `hops` links."""
    parts, i, cur = path.split("/"), 0, ""
    while i < len(parts):
        nxt = parts[i] if not cur else cur + "/" + parts[i]
        m = final.get(nxt)
        if m is not None and m.issym():
            hops -= 1
            if hops < 0 or m.linkname.startswith("/"):
                return None
            path = posixpath.normpath(posixpath.join(posixpath.dirname(nxt), m.linkname, *parts[i + 1:]))
            if _leaves(path):
                return None
            parts, i, cur = path.split("/"), 0, ""
            continue
        cur, i = nxt, i + 1
    return final.get(cur), hops


def select_members(members):
    """What the reference's `find -name "*.so" | xargs strip` changes in the tree tarfile extracts from `members`:
    (sorted indexes of the regular members whose data it strips, the number of `*.so` entries it leaves alone).

    A regular member named *.so is stripped.  A hard link named *.so strips the last regular member of its linkname
    before it, and a symlink named *.so the regular member it resolves to (relative to the link's directory, through
    up to 40 symlink members): GNU strip writes through a link into the target's inode.  Directories, sparse members,
    dangling links and links that leave the archive are left alone."""
    index = {id(m): i for i, m in enumerate(members)}
    final = {}
    for m in members:
        final[_norm(m.name)] = m

    def target(m, pos, hops):
        while hops >= 0:
            if m.isreg():
                return None if m.issparse() else index[id(m)]
            if m.islnk():
                name, m = _norm(m.linkname), None
                for k in range(pos - 1, -1, -1):
                    if _norm(members[k].name) == name:
                        m, pos = members[k], k
                        break
                if m is None:
                    return None
                hops -= 1
                continue
            if m.issym():
                path = posixpath.normpath(posixpath.join(posixpath.dirname(_norm(m.name)), m.linkname))
                if m.linkname.startswith("/") or _leaves(path):
                    return None
                r = _resolve(path, final, hops - 1)
                if r is None or r[0] is None:
                    return None
                m, hops = r
                pos = index[id(m)]
                continue
            return None
        return None

    chosen, skipped = set(), 0
    for i, m in enumerate(members):
        if not posixpath.basename(m.name).endswith(".so"):
            continue
        t = target(m, i, _SYMLINK_HOPS)
        if t is None:
            skipped += 1
        else:
            chosen.add(t)
    return sorted(chosen), skipped


def _pax_record(keyword, value):
    """one pax record, its length prefix computed as TarInfo._create_pax_generic_header computes it"""
    n = len(keyword) + len(value) + 3
    p = 0
    while True:
        q = n + len(str(p))
        if q == p:
            break
        p = q
    return str(p).encode("ascii") + b" " + keyword + b"=" + value + b"\n"


def _sealed(block, size):
    """a header block with its size field and checksum rewritten as tarfile writes them"""
    b = bytearray(block)
    b[124:136] = tarfile.itn(size, 12, tarfile.GNU_FORMAT)
    b[148:156] = b"%06o\0 " % tarfile.calc_chksums(bytes(b))[0]
    return bytes(b)


def _pax_records(buf):
    """the records of a pax header's data, framed as _proc_pax frames them: [(record bytes, keyword)]"""
    out, pos = [], 0
    while pos < len(buf) and buf[pos] != 0:
        sp = buf.index(b" ", pos)
        length = int(buf[pos:sp])
        rec = buf[pos:pos + length]
        out.append((rec, rec[sp - pos + 1:].split(b"=", 1)[0]))
        pos += length
    return out


def rewrite_headers(chain, size):
    """The header blocks of a member (`chain`: from TarInfo.offset to offset_data) for its data replaced by `size`
    bytes: the size field and checksum of the member's header, and the `size` record of a pax `x` header in front
    of it with that header's size, checksum and padding."""
    out, pos = bytearray(), 0
    while pos < len(chain):
        h = chain[pos:pos + BLOCKSIZE]
        t = h[156:157]
        if t in (tarfile.GNUTYPE_LONGNAME, tarfile.GNUTYPE_LONGLINK, tarfile.XHDTYPE, tarfile.XGLTYPE,
                 tarfile.SOLARIS_XHDTYPE):
            n = tarfile.nti(h[124:136])
            data = chain[pos + BLOCKSIZE:pos + BLOCKSIZE + n]
            blocks = -(-n // BLOCKSIZE) * BLOCKSIZE
            recs = _pax_records(data) if t in (tarfile.XHDTYPE, tarfile.SOLARIS_XHDTYPE) else []
            if any(k == b"size" for _, k in recs):
                data = b"".join(_pax_record(b"size", b"%d" % size) if k == b"size" else r for r, k in recs)
                out += _sealed(h, len(data)) + data + bytes(-len(data) % BLOCKSIZE)
            else:
                out += chain[pos:pos + BLOCKSIZE + blocks]
            pos += BLOCKSIZE + blocks
            continue
        out += _sealed(h, size) + chain[pos + BLOCKSIZE:]
        break
    return bytes(out)


def _pieces(segs, piece):
    """segments [(address, length)] cut into pieces of exactly `piece` bytes, the last one shorter"""
    cur, fill = [], 0
    for addr, k in segs:
        while k:
            t = min(k, piece - fill)
            cur.append((addr, t))
            addr, k, fill = addr + t, k - t, fill + t
            if fill == piece:
                yield cur
                cur, fill = [], 0
    if cur:
        yield cur


def strip_with(src, dst, reader, indexer, stripper, open_writer, piece_bytes=PIECE_BYTES, fallback_host_strip=True,
               tolerate_non_elf=False):
    """strip_tarball with the engines given (GpuTarReader, GpuTarIndex, zipfile_gpu.GpuStripper and
    open_writer(fileobj, name, mtime) -> a GpuGzipFile fed by submit_device, or stand-ins with the same interfaces)."""
    from .zipfile_gpu import StripFailed, _umask
    src, dst = os.fspath(src), os.fspath(dst)
    if os.path.realpath(src) == os.path.realpath(dst) or (os.path.exists(dst) and os.path.samefile(src, dst)):
        raise ValueError("strip_tarball: %r is the archive being read; write the result somewhere else" % dst)
    if piece_bytes < 1:
        raise ValueError("pieces of %d bytes" % piece_bytes)
    out_dir = os.path.dirname(dst) or "."
    os.makedirs(out_dir, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix=os.path.basename(dst) + ".", suffix=".tmp", dir=out_dir)
    try:
        with os.fdopen(fd, "wb") as fp:
            (base, n), mtime = reader.read(src)
            members, stop, view, (ranges, data, ist) = list_members((base, n), indexer, reader)
            chosen, skipped = select_members(members)
            res = stripper.strip([(base + members[i].offset_data, members[i].size) for i in chosen]) if chosen else []
            new, c = {}, {"gpu": 0, "fallback": 0, "skipped": skipped, "in_bytes": 0, "out_bytes": 0}
            for i, (status, ref) in zip(chosen, res):
                m = members[i]
                if status == N.ST_OK:
                    c["gpu"] += 1
                elif status == N.ST_NOT_ELF and tolerate_non_elf:
                    c["skipped"] += 1
                    continue
                else:
                    old = stripper.fetch((base + m.offset_data, m.size))
                    fixed = stripper.host_strip(old) if fallback_host_strip else None
                    if fixed is None:
                        if tolerate_non_elf and old[:4] != b"\x7fELF":
                            c["skipped"] += 1
                            continue
                        raise StripFailed(m.name, "strip refuses this file (the reference's xargs exits 123)"
                                          if fallback_host_strip else "not stripped on the GPU, and the host strip is off")
                    c["fallback"] += 1
                    ref = stripper.upload(fixed)
                new[i] = ref
                c["in_bytes"] += m.size
                c["out_bytes"] += ref[1]
            # the new tar stream: unchanged runs of the source, rewritten headers, stripped files, zero padding
            plan, staging, pos = [], bytearray(), 0
            for i in sorted(new):
                m = members[i]
                plan.append(("src", pos, m.offset - pos))
                view.seek(m.offset)
                head = rewrite_headers(view.read(m.offset_data - m.offset), new[i][1])
                plan.append(("hdr", len(staging), len(head)))
                staging += head
                plan.append(("dev", new[i][0], new[i][1]))
                plan.append(("zero", 0, -new[i][1] % BLOCKSIZE))
                pos = m.offset_data + -(-m.size // BLOCKSIZE) * BLOCKSIZE
            plan.append(("src", pos, stop - pos))
            body = sum(k for _, _, k in plan)
            plan.append(("zero", 0, 2 * BLOCKSIZE + -(body + 2 * BLOCKSIZE) % RECORDSIZE))
            d_head = reader.upload(staging) if staging else 0
            d_zero = reader.zeros(RECORDSIZE)
            segs = []
            for kind, at, k in plan:
                while k > 0:
                    t = min(k, RECORDSIZE) if kind == "zero" else k
                    addr = {"src": base + at, "hdr": d_head + at, "dev": at, "zero": d_zero}[kind]
                    if segs and kind == "src" and segs[-1][0] + segs[-1][1] == addr:
                        segs[-1] = (segs[-1][0], segs[-1][1] + t)
                    else:
                        segs.append((addr, t))
                    k -= t
            tar_out = sum(k for _, k in segs)
            gz = open_writer(fp, dst, mtime)
            try:
                for piece in _pieces(segs, piece_bytes):
                    gz.submit_device(piece)
            finally:
                gz.close()
            dst_bytes = fp.tell()
        os.chmod(tmp, 0o666 & ~_umask())
        os.replace(tmp, dst)
    except BaseException:
        os.unlink(tmp)
        raise
    deflate = dict(gz.stats or {})
    deflated = max(deflate.get("out_bytes", 2) - 2, 0)   # the final block's 2 bytes are written on the host
    index = dict(ist, ranges=len(ranges), bytes=len(data), misses=view.misses, miss_bytes=view.miss_bytes)
    st = {"members": len(members), "selected": len(chosen), "gpu": c["gpu"], "fallback": c["fallback"],
          "skipped": c["skipped"], "in_bytes": c["in_bytes"], "out_bytes": c["out_bytes"],
          "tar_bytes_in": n, "tar_bytes_out": tar_out, "src_bytes": os.path.getsize(src), "dst_bytes": dst_bytes,
          "uploaded_bytes": reader.uploaded + stripper.uploaded,
          "downloaded_bytes": reader.downloaded + 16 * len(ranges) + len(data) + deflated + stripper.downloaded,
          "index": index, "inflate": reader.stats(), "strip": stripper.stats(), "deflate": deflate}
    st["kernel_ms"] = (st["inflate"].get("kernel_ms", 0.0) + index.get("kernel_ms", 0.0) + sum(st["strip"].values()) +
                       deflate.get("deflate_ms", 0.0) + deflate.get("crc_ms", 0.0) + deflate.get("h2d_ms", 0.0))
    return st


def strip_tarball(src, dst, ctx=None, compresslevel=None, fallback_host_strip=True, tolerate_non_elf=False,
                  piece_bytes=PIECE_BYTES, seek_table=False):
    """Write `dst` as `src` (a .tar.gz) with every shared object stripped: the tar stream the reference's three passes
    (tarfile "r:gz" extract, `find -name "*.so" | xargs strip`, tarfile "w:gz") would write, without the tree.

    The gzip file is uploaded once and inflated on the GPU; the tar stream stays in device memory, where one warp
    walks its headers (lb2_tar_index) so that tarfile lists the members from a single download; the selected members
    (select_members) are stripped where they lie (lb2_strip_device_async) and the new tar stream -- unchanged runs of
    the source, rewritten headers, stripped files and zero padding -- is deflated straight from device memory
    (lb2_gzip_submit_device).  Only compressed bytes and the headers cross the bus.

    The tar stream of dst: every member in source order keeps its header blocks byte for byte except, for a stripped
    member, its size field (tarfile.itn), its checksum ("%06o\\0 ") and the `size` record of a pax header in front of
    it; stripped data is zero-padded to 512 bytes; two zero blocks and zero padding to a multiple of RECORDSIZE end
    it, as TarFile.close() writes them; nothing after the source's end-of-archive marker is kept.  The gzip layer is
    one member with GpuGzipFile's header (MTIME from the source's first member) and the DEFLATE body GpuGzipFile
    writes for that tar stream at the same compresslevel and piece_bytes; seek_table=True appends GpuGzipFile's seek
    table, so that dst reads back in one pass.  A source with a seek table is read from it.

    An ELF the planner refuses is fetched, stripped by the host `strip` and uploaded again (fallback_host_strip); a
    member `strip` refuses raises zipfile_gpu.StripFailed unless it is not an ELF and tolerate_non_elf keeps it.
    Framing, data and trailer errors raise what gunzip raises, the member headers what tarfile raises, and a tar
    stream that does not fit on the device NativeError(LB2_E_CAPACITY).  dst appears when it is complete and not at
    all when the call raises; dst == src raises ValueError.

    Returns a stats dict: members, selected, gpu, fallback, skipped; in_bytes / out_bytes (the stripped members before
    and after); tar_bytes_in / tar_bytes_out; src_bytes / dst_bytes; uploaded_bytes / downloaded_bytes (everything
    that crossed the bus); index (the walk's stats, ranges, bytes and misses), inflate, strip and deflate (the
    engines' stats) and kernel_ms, their kernel times summed.  There is no CPU path: without a GPU this raises."""
    from .zipfile_gpu import GpuStripper
    N.deflate_flags(compresslevel)
    own = False
    if ctx is None:
        ctx, own = _default_context()

    def open_writer(fileobj, name, mtime):
        return GpuGzipFile(name, mtime=mtime, ctx=ctx, piece_bytes=piece_bytes, compresslevel=compresslevel,
                           fileobj=fileobj, host_buffers=False, seek_table=seek_table)
    try:
        with GpuTarReader(ctx) as reader, GpuStripper(ctx) as stripper:
            return strip_with(src, dst, reader, GpuTarIndex(ctx), stripper, open_writer, piece_bytes,
                              fallback_host_strip, tolerate_non_elf)
    finally:
        if own:
            ctx.close()


def main(argv=None):
    """python -m lambdipy_b200.tarball strip SRC DST [--level 9] [--seek-table]"""
    import argparse
    ap = argparse.ArgumentParser(prog="python -m lambdipy_b200.tarball")
    sub = ap.add_subparsers(dest="command", required=True)
    sp = sub.add_parser("strip", help="strip the *.so members of the .tar.gz SRC on the GPU and write the result to DST")
    sp.add_argument("src")
    sp.add_argument("dst")
    sp.add_argument("--level", type=int, choices=[9], default=None, help="9: the optimal parse (smaller, slower)")
    sp.add_argument("--seek-table", action="store_true",
                    help="append a seek table, with which the GPU reader decodes DST without searching for block starts")
    args = ap.parse_args(argv)
    st = strip_tarball(args.src, args.dst, compresslevel=args.level, **ST.seek_kw(args.seek_table))
    print("Tarball: %s, %.1f MB -> %.1f MB; %d shared objects stripped (%d via host strip), %.1f MB -> %.1f MB"
          % (args.dst, st["src_bytes"] / 1e6, st["dst_bytes"] / 1e6, st["gpu"] + st["fallback"], st["fallback"],
             st["in_bytes"] / 1e6, st["out_bytes"] / 1e6))
    return 0


if __name__ == "__main__":
    import sys
    sys.exit(main())
