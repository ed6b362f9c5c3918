"""Lambda deployment zips with every member's DEFLATE body compressed on the GPU, and zips read back on the GPU.

A zip is the only package format AWS Lambda accepts, so the last step after `lambdipy build` is zipping `./build`,
usually with `shutil.make_archive` or `zip -r`: zlib on one core over the whole bundle.

    zip_tree(root_dir, zip_path)     writes what `shutil.make_archive(zip_path[:-4], "zip", root_dir)` writes under
                                     Python 3.12 -- the same walk (os.walk, sorted directories, files in scandir
                                     order, symlinks followed), the same entries in the same order with the same
                                     names, times, attributes, versions, flag bits and (zip64) headers -- except for
                                     the member bodies, their compressed sizes and the header offsets that follow.

Every file is ZIP_DEFLATED and every directory ZIP_STORED, as in make_archive.  The bodies come from the CUDA encoder
behind `lb2_zip_*` (csrc/deflate.cu): each member is its own raw DEFLATE stream (64 KB chunks, sync-flushed, closed
by the final block 03 00; an empty file's body is exactly 03 00, as zlib's), and its CRC-32 is computed on the GPU.
Files are packed into two pinned pieces in flight, so reading the files overlaps the kernels; a file that goes on
into the next piece is cut at a multiple of 64 KB of its bytes, so it is deflated in the chunks of the whole file.

The container is written here, with the standard library's `ZipInfo` for every local header.  The seam between the
two is the encoder (`GpuZipEncoder`): anything with the same `buffers` / `submit` / `collect` can stand in for it.

    extract_zip(zip_path, directory)  the tree `ZipFile(zip_path).extractall(directory)` writes
    testzip(zip_path)                 the first bad member's name or None, as `ZipFile(zip_path).testzip()`

read every STORED and DEFLATE member with the CUDA decoder behind `lb2_unzip_*` (csrc/inflate.cu): all members of a
batch are inflated and CRC-checked in one pass, each bounded by its own body.  The seam there is the decoder
(`GpuUnzipDecoder`).

    strip_zip(src_zip, dst_zip)       the zip `extractall`, the reference's `find -name "*.so" | xargs strip` and
                                      `make_archive` would make of src_zip, members and order kept

chains the three engines on the device: the `*.so` members are inflated by the decoder, stripped where they lie by
the strip kernels (`GpuStripper`) and deflated by the encoder straight from the stripped arena
(`lb2_zip_submit_device`); every other member's body is copied from src_zip as it is.
`python -m lambdipy_b200.zipfile_gpu strip SRC DST [--level 9]` is the same call from a shell.
"""
import copy
import ctypes as C
import os
import struct
import subprocess
import sys
import tempfile
import zipfile

from . import _native as N
from . import seek_table as ST
from .seek_table import seek_kw

PIECE_BYTES = 64 << 20  # file bytes (and padding) per GPU submission
MAX_SEGS = 1 << 16      # files per piece
ALIGN = 16              # each file starts at a 16-byte-aligned offset of its piece (the CRC kernel's vector loads)
CHUNK = 65536           # the encoder's chunk (GZ_CHUNK): a file continued in the next piece is cut at a multiple of it


class GpuZipEncoder:
    """The lb2_zip_* writer with its two pinned piece buffers.

    buffers[k]: writable memoryview of piece_bytes; submit(k, n, seg_off, seg_len, flags) hands buffers[k][:n] to the
    GPU (flags: N.ZIP_CONTINUES / N.ZIP_MORE); collect() waits for the oldest piece and returns (its DEFLATE bytes,
    [(out_off, out_len, crc32, ended) per segment]); the bytes stay valid until the next collect().
    compresslevel: None (the default encoder) or 9 (the optimal parse, LB2_DEFLATE_BEST).

    submit_device(refs, flags) hands over a piece whose segments are (device address, length) pairs instead, laid out
    by the library (lb2_zip_submit_device); a writer fed only that way needs no piece buffers (host_buffers=False).

    seek_table=True: after each collect(), seek_chunks holds every segment's [(compressed, decoded)] 64 KB chunks
    (lb2_zip_chunk_sizes), from which the container writes each member's seek table (seek_table.py); else it is None."""

    def __init__(self, ctx, piece_bytes=PIECE_BYTES, max_segs=MAX_SEGS, compresslevel=None, host_buffers=True,
                 seek_table=False):
        flags = N.deflate_flags(compresslevel)  # checked before anything is allocated
        self._ctx, self._z, self._ptrs, self._out = ctx, None, [], None
        self.piece_bytes, self.max_segs = int(piece_bytes), int(max_segs)
        try:
            z = C.c_void_p()
            ctx.check(ctx.lib.lb2_zip_create(ctx.h, flags, C.byref(z)))
            self._z = z
            self.buffers = []
            for _ in range(2 if host_buffers else 0):
                p = ctx.pinned_alloc(self.piece_bytes)
                self._ptrs.append(p)
                self.buffers.append(memoryview((C.c_uint8 * self.piece_bytes).from_address(p)).cast("B"))
            self._cap = N.zip_bound(self.piece_bytes, self.max_segs)
            self._out = ctx.pinned_alloc(self._cap)
        except BaseException:
            self.close()
            raise
        self._pending = []  # segment lengths of each piece in flight
        self._stats = N.GzipStats()
        self._seek = bool(seek_table)
        self.seek_chunks = None

    def submit(self, k, n, seg_off, seg_len, flags):
        ns = len(seg_off)
        offs, lens = (C.c_uint64 * ns)(*seg_off), (C.c_uint64 * ns)(*seg_len)
        self._ctx.check(self._ctx.lib.lb2_zip_submit(self._z, self._ptrs[k], n, offs, lens, ns, flags))
        self._pending.append(list(seg_len))

    def submit_device(self, refs, flags):
        ns = len(refs)
        src = (N.ZipSource * ns)()
        for i, (addr, n) in enumerate(refs):
            src[i].d_ptr, src[i].len = addr, n
        self._ctx.check(self._ctx.lib.lb2_zip_submit_device(self._z, src, ns, flags))
        self._pending.append([n for _, n in refs])

    def collect(self):
        lens = self._pending.pop(0)
        ns = len(lens)
        segs, n = (N.ZipSegment * ns)(), C.c_uint64()
        self._ctx.check(self._ctx.lib.lb2_zip_collect(self._z, self._out, self._cap, C.byref(n), segs, C.byref(self._stats)))
        body = memoryview((C.c_uint8 * n.value).from_address(self._out)).cast("B") if n.value else memoryview(b"")
        if self._seek:
            counts = [max(1, -(-k // CHUNK)) for k in lens]
            sizes, k = (C.c_uint32 * max(sum(counts), 1))(), C.c_uint32()
            self._ctx.check(self._ctx.lib.lb2_zip_chunk_sizes(self._z, sizes, len(sizes), C.byref(k)))
            if k.value != sum(counts):
                raise RuntimeError("lb2_zip_chunk_sizes: %d chunks for %d" % (k.value, sum(counts)))
            self.seek_chunks, at = [], 0
            for seg, length, cnt in zip(segs, lens, counts):
                ch = [(sizes[at + j], min(CHUNK, length - j * CHUNK)) for j in range(cnt)]
                if sum(c for c, _ in ch) != seg.out_len:
                    raise RuntimeError("lb2_zip_chunk_sizes: the chunks of a segment do not add up to its bytes")
                self.seek_chunks.append(ch)
                at += cnt
        return body, [(s.out_off, s.out_len, s.crc32, bool(s.ended)) for s in segs]

    def stats(self):
        st = self._stats
        return {"kernel_ms": st.deflate_ms + st.crc_ms, "deflate_ms": st.deflate_ms, "crc_ms": st.crc_ms,
                "h2d_ms": st.h2d_ms, "d2h_ms": st.d2h_ms, "n_chunks": st.n_chunks,
                "n_stored_chunks": st.n_stored_chunks, "n_fixed_chunks": st.n_fixed_chunks,
                "n_opt_chunks": st.n_opt_chunks, "best_ms": st.best_ms}

    def close(self):
        if self._z is not None:
            self._ctx.lib.lb2_zip_destroy(self._z)
            self._z = None
        self.buffers = []
        for p in self._ptrs:
            self._ctx.pinned_free(p)
        self._ptrs = []
        if self._out is not None:
            self._ctx.pinned_free(self._out)
            self._out = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def tree_entries(root_dir):
    """(path, ZipInfo) of every entry `shutil.make_archive(base, "zip", root_dir)` writes, in its order."""
    entries = []
    for dirpath, dirnames, filenames in os.walk(os.path.normpath(os.path.join(root_dir, os.curdir))):
        arcdir = os.path.normpath(os.path.relpath(dirpath, root_dir))
        for name in sorted(dirnames):
            path = os.path.join(dirpath, name)
            entries.append((path, zipfile.ZipInfo.from_file(path, os.path.join(arcdir, name))))
        for name in filenames:
            path = os.path.normpath(os.path.join(dirpath, name))
            if os.path.isfile(path):
                entries.append((path, zipfile.ZipInfo.from_file(path, os.path.join(arcdir, name))))
    return entries


def central_directory(infos, start, comment=b"", tables=None):
    """The central directory of `infos` (written from offset `start`) and the end records, as ZipFile.close() writes
    them: zip64 extras for sizes or offsets beyond ZIP64_LIMIT, zip64 end records beyond 65 535 entries or 4 GiB, then
    the archive comment.  tables {index: seek table}: appended to that entry's extra fields, either a member's
    [(compressed, decoded)] chunks (seek_table.zip_field) or a field kept as it is."""
    out = []
    for i, zi in enumerate(infos):
        dt = zi.date_time
        dosdate = (dt[0] - 1980) << 9 | dt[1] << 5 | dt[2]
        dostime = dt[3] << 11 | dt[4] << 5 | (dt[5] // 2)
        extra = []
        if zi.file_size > zipfile.ZIP64_LIMIT or zi.compress_size > zipfile.ZIP64_LIMIT:
            extra += [zi.file_size, zi.compress_size]
            file_size = compress_size = 0xFFFFFFFF
        else:
            file_size, compress_size = zi.file_size, zi.compress_size
        if zi.header_offset > zipfile.ZIP64_LIMIT:
            extra.append(zi.header_offset)
            header_offset = 0xFFFFFFFF
        else:
            header_offset = zi.header_offset
        extra_data, min_version = zi.extra, 0
        if extra:
            extra_data = zipfile._strip_extra(extra_data, (1,))
            extra_data = struct.pack("<HH" + "Q" * len(extra), 1, 8 * len(extra), *extra) + extra_data
            min_version = zipfile.ZIP64_VERSION
        t = tables.get(i) if tables else None
        if t is not None:
            extra_data += t if isinstance(t, bytes) else ST.zip_field(t, len(extra_data))
        filename, flag_bits = zi._encodeFilenameFlags()
        out.append(struct.pack(zipfile.structCentralDir, zipfile.stringCentralDir, max(min_version, zi.create_version),
                               zi.create_system, max(min_version, zi.extract_version), zi.reserved, flag_bits,
                               zi.compress_type, dostime, dosdate, zi.CRC, compress_size, file_size, len(filename),
                               len(extra_data), len(zi.comment), 0, zi.internal_attr, zi.external_attr, header_offset))
        out += [filename, extra_data, zi.comment]
    cd = b"".join(out)
    count, size, offset = len(infos), len(cd), start
    if count > zipfile.ZIP_FILECOUNT_LIMIT or offset > zipfile.ZIP64_LIMIT or size > zipfile.ZIP64_LIMIT:
        cd += struct.pack(zipfile.structEndArchive64, zipfile.stringEndArchive64, zipfile.sizeEndCentDir64 - 12, 45, 45,
                          0, 0, count, count, size, offset)
        cd += struct.pack(zipfile.structEndArchive64Locator, zipfile.stringEndArchive64Locator, 0, start + size, 1)
        count, size, offset = min(count, 0xFFFF), min(size, 0xFFFFFFFF), min(offset, 0xFFFFFFFF)
    return cd + struct.pack(zipfile.structEndArchive, zipfile.stringEndArchive, 0, 0, count, count, size, offset,
                            len(comment)) + comment


class _ContainerWriter:
    """Writes the entries in order as their bodies arrive: a directory as soon as every entry before it is written;
    a file's local header when its first body bytes arrive, rewritten with the CRC and sizes once it ends (seeking
    back, as ZipFile does on a seekable file).  With `copy` (strip_zip), an entry whose body never arrives is not a
    directory of the tree but a member kept as it is: copy(ZipInfo) writes its header and body at the current
    position.  part(..., chunks) with every part's chunks gives the file a seek table in the central directory;
    tables {entry index: table} are what central_directory writes."""

    def __init__(self, fp, entries, copy=None):
        self.fp, self.entries, self.next, self.copy = fp, entries, 0, copy
        self.cur = None  # (ZipInfo, zip64) of the file being written
        self.tables = {}
        self.in_bytes = self.out_bytes = self.n_files = 0

    def _upto(self, idx):
        while self.next < idx:
            zi = self.entries[self.next][1]
            zi.header_offset = self.fp.tell()
            if self.copy is not None:
                self.copy(zi)
            else:
                assert zi.is_dir(), "file entry %s written out of order" % zi.filename
                zi.compress_size = zi.CRC = 0
                self.fp.write(zi.FileHeader(False))
            self.next += 1

    def part(self, idx, body, crc, ended, file_bytes, chunks=None):
        if self.cur is None:
            self._upto(idx)
            zi = self.entries[idx][1]
            zi.compress_type = zipfile.ZIP_DEFLATED
            zi.compress_size = zi.CRC = 0
            zi.flag_bits = 0
            if not zi.external_attr:
                zi.external_attr = 0o600 << 16
            zip64 = zi.file_size * 1.05 > zipfile.ZIP64_LIMIT  # ZipFile's guess from the size at stat time
            zi.header_offset = self.fp.tell()
            self.fp.write(zi.FileHeader(zip64))
            self.cur, self.cur_in, self.cur_out = (zi, zip64), 0, 0
            self.cur_chunks = []
        self.fp.write(body)
        self.cur_chunks = None if chunks is None or self.cur_chunks is None else self.cur_chunks + chunks
        self.cur_in += file_bytes
        self.cur_out += len(body)
        if ended:
            zi, zip64 = self.cur
            zi.CRC, zi.file_size, zi.compress_size = crc, self.cur_in, self.cur_out
            if not zip64 and (zi.file_size > zipfile.ZIP64_LIMIT or zi.compress_size > zipfile.ZIP64_LIMIT):
                raise RuntimeError("%s: file size grew past 4 GiB while it was zipped" % zi.filename)
            end = self.fp.tell()
            self.fp.seek(zi.header_offset)
            self.fp.write(zi.FileHeader(zip64))
            self.fp.seek(end)
            self.in_bytes += self.cur_in
            self.out_bytes += self.cur_out
            self.n_files += 1
            self.tables.pop(idx, None)
            if self.cur_chunks:
                self.tables[idx] = self.cur_chunks
            self.cur = None
            self.next = idx + 1

    def finish(self, comment=b""):
        self._upto(len(self.entries))
        start = self.fp.tell()
        self.fp.write(central_directory([zi for _, zi in self.entries], start, comment, self.tables))


def _read_into(f, view):
    got = 0
    while got < len(view):
        k = f.readinto(view[got:])
        if not k:
            break
        got += k
    return got


def write_zip(root_dir, zip_path, encoder):
    """zip_tree with the member bodies from `encoder` (GpuZipEncoder, or a stand-in with the same interface).
    Returns the stats dict of zip_tree."""
    archive_dir = os.path.dirname(zip_path)
    if archive_dir and not os.path.exists(archive_dir):
        os.makedirs(archive_dir)
    piece, max_segs = len(encoder.buffers[0]), encoder.max_segs
    if piece < CHUNK:
        raise ValueError("pieces of %d bytes: at least %d are needed" % (piece, CHUNK))
    with open(zip_path, "w+b") as fp:
        entries = tree_entries(root_dir)
        w = _ContainerWriter(fp, entries)
        in_flight = []                    # per piece: [(entry index, bytes)] of its segments
        k, fill, segs, cont = 0, 0, [], False

        def collect():
            body, res = encoder.collect()
            chunks = getattr(encoder, "seek_chunks", None) or [None] * len(res)
            for (idx, nbytes), (off, n, crc, ended), ch in zip(in_flight.pop(0), res, chunks):
                w.part(idx, body[off:off + n], crc, ended, nbytes, ch)

        def submit(more):
            nonlocal k, fill, segs, cont
            flags = (N.ZIP_CONTINUES if cont else 0) | (N.ZIP_MORE if more else 0)
            encoder.submit(k, fill, [s[1] for s in segs], [s[2] for s in segs], flags)
            in_flight.append([(s[0], s[2]) for s in segs])
            k, fill, segs, cont = k ^ 1, 0, [], more
            if len(in_flight) == 2:  # the buffer to fill next belongs to the older piece: wait for it
                collect()

        for idx, (path, zi) in enumerate(entries):
            if zi.is_dir():
                continue
            with open(path, "rb") as f:
                remaining = zi.file_size
                while True:
                    # A file that does not fit in the rest of the piece is cut at a multiple of CHUNK of its own bytes,
                    # so its chunks fall where they would if it were deflated whole: a cut elsewhere would cost one
                    # more chunk (and its stored-block and sync-flush framing) per piece boundary.
                    off = -(-fill // ALIGN) * ALIGN
                    if len(segs) == max_segs or off > piece or (remaining > piece - off and piece - off < CHUNK):
                        submit(False)
                        off = 0
                    want = remaining if remaining <= piece - off else (piece - off) // CHUNK * CHUNK
                    got = _read_into(f, encoder.buffers[k][off:off + want])
                    segs.append((idx, off, got))
                    fill = off + got
                    remaining -= got
                    if got < want or not remaining:  # the end of the file (or it shrank since it was listed)
                        break
                    submit(True)                     # the piece is full and the file goes on in the next one
        if segs:
            submit(False)
        while in_flight:
            collect()
        w.finish()
        zip_bytes = fp.tell()
    st = {"files": w.n_files, "entries": len(entries), "in_bytes": w.in_bytes, "out_bytes": w.out_bytes,
          "zip_bytes": zip_bytes}
    st.update(encoder.stats())
    return st


def zip_tree(root_dir, zip_path, ctx=None, piece_bytes=PIECE_BYTES, compresslevel=None, seek_table=False):
    """Write `zip_path` as `shutil.make_archive(zip_path[:-4], "zip", root_dir)` would, with every member's DEFLATE
    body and CRC-32 computed on the GPU.  Returns a stats dict: files, entries, in_bytes (file bytes), out_bytes
    (member bodies), zip_bytes, kernel_ms (deflate + CRC-32 kernels, CUDA events), n_chunks, n_stored_chunks,
    n_fixed_chunks, n_opt_chunks and the copy times.  ctx=None: the context the strip path has already warmed up, if
    any, else a new one on device LAMBDIPY_B200_DEVICE (default 0).  compresslevel: None keeps the default encoder,
    9 selects the optimal parse (smaller, slower); anything else raises ValueError.  seek_table=True gives every
    DEFLATE member of two or more 64 KB chunks a seek table in its central-directory entry (seek_table.py), with which
    the GPU reader decodes it without searching for block starts; the archive up to the central directory is the one
    written without.  There is no CPU path: without a GPU this raises."""
    from .tarball import _default_context
    N.deflate_flags(compresslevel)
    own = False
    if ctx is None:
        ctx, own = _default_context()
    try:
        with GpuZipEncoder(ctx, piece_bytes, compresslevel=compresslevel, seek_table=seek_table) as enc:
            return write_zip(root_dir, zip_path, enc)
    finally:
        if own:
            ctx.close()


# ---- reading: extract_zip / testzip ------------------------------------------------------------------------------
# The central directory is parsed by the standard library (zip64, a prepended offset and data descriptors included);
# each member's local header is read from the uploaded buffer to find its body, and every member the GPU can take is
# decoded and CRC-checked by lb2_unzip_run.  The seam is the decoder (`GpuUnzipDecoder`): anything with the same
# `buffer` / `run` / `stats` can stand in for it.

BATCH_BYTES = 1 << 30   # archive bytes plus 3 bytes per output byte of one batch (the device memory it needs, at most)
UNZIP_OK, UNZIP_BAD_DATA, UNZIP_WRONG_SIZE, UNZIP_BAD_CRC = 0, 1, 2, 3
_GPU_METHODS = (zipfile.ZIP_STORED, zipfile.ZIP_DEFLATED)
_STDLIB_FLAGS = 0x1 | 0x20 | 0x40   # encrypted, compressed patched data, strong encryption: the stdlib's own code


class BadZipMember(zipfile.BadZipFile):
    """A member whose DEFLATE data is invalid or truncated, or that decodes to another size than the archive records."""

    def __init__(self, name, why):
        super().__init__("%s for file %r" % (why, name))
        self.member = name


class DeviceTooSmall(Exception):
    """The batch does not fit in device memory (lb2_unzip_run returned LB2_E_CAPACITY)."""


class GpuUnzipDecoder:
    """The lb2_unzip_* reader with a pinned input and output buffer.

    buffer(n): a writable memoryview of n bytes, valid until the next buffer(); run(n, members) decodes
    members [(body_off, body_len, size, crc32, method)] of buffer[:n] and returns [(status, data)] with status one of
    UNZIP_* and data a memoryview of the member's bytes, valid until the next run(); DeviceTooSmall when the batch
    does not fit on the device."""

    def __init__(self, ctx):
        self._ctx, self._u, self._in, self._out = ctx, None, None, None
        self._in_cap = self._out_cap = 0
        u = C.c_void_p()
        ctx.check(ctx.lib.lb2_unzip_create(ctx.h, 0, C.byref(u)))
        self._u = u
        self._stats = {}

    def _grow(self, attr, need):
        cap = getattr(self, attr + "_cap")
        if need <= cap:
            return getattr(self, attr)
        if getattr(self, attr) is not None:
            self._ctx.pinned_free(getattr(self, attr))
            setattr(self, attr, None)
            setattr(self, attr + "_cap", 0)
        cap = max(need, 2 * cap, 1 << 20)
        setattr(self, attr, self._ctx.pinned_alloc(cap))
        setattr(self, attr + "_cap", cap)
        return getattr(self, attr)

    def buffer(self, n):
        p = self._grow("_in", n)
        return memoryview((C.c_uint8 * n).from_address(p)).cast("B") if n else memoryview(bytearray())

    def run(self, n, members, device=False, tables=None):
        """tables (may be None): one seek table [(compressed, decoded)] or None per member (lb2_unzip_run_table)"""
        k = len(members)
        tab = (N.UnzipMember * max(k, 1))()
        for i, (off, blen, size, crc, method) in enumerate(members):
            tab[i].body_off, tab[i].body_len, tab[i].size, tab[i].crc32, tab[i].method = off, blen, size, crc, method
        res, out_n, st = (N.UnzipResult * max(k, 1))(), C.c_uint64(), N.UnzipStats()
        lib = self._ctx.lib
        if tables:
            first = (C.c_uint32 * (k + 1))()
            flat = [e for t in tables for e in (t or [])]
            spans = (N.InflateSpan * max(len(flat), 1))()
            for i, t in enumerate(tables):
                first[i + 1] = first[i] + len(t or [])
            for i, (c, u) in enumerate(flat):
                spans[i].in_len, spans[i].out_len = c, u
            used, refused = C.c_uint32(), C.c_uint32()
            rc = lib.lb2_unzip_run_table(self._u, self._in if n else None, n, tab, k, first, spans, C.byref(out_n), res,
                                         C.byref(st), C.byref(used), C.byref(refused))
            self._stats["seek_table"] = self._stats.get("seek_table", 0) + used.value
            self._stats["seek_table_refused"] = self._stats.get("seek_table_refused", 0) + refused.value
        else:
            rc = lib.lb2_unzip_run(self._u, self._in if n else None, n, tab, k, C.byref(out_n), res, C.byref(st))
        if rc == N.LB2_E_CAPACITY:
            raise DeviceTooSmall((lib.lb2_last_error(self._ctx.h) or b"").decode())
        self._ctx.check(rc)
        for key, v in st.as_dict().items():
            self._stats[key] = self._stats.get(key, 0) + v
        if device:
            d_out, d_n = C.c_void_p(), C.c_uint64()
            self._ctx.check(lib.lb2_unzip_device_output(self._u, C.byref(d_out), C.byref(d_n)))
            return [(res[i].status, ((d_out.value or 0) + res[i].out_off, members[i][2])) for i in range(k)]
        p = self._grow("_out", out_n.value)
        self._ctx.check(lib.lb2_unzip_read(self._u, p, out_n.value))
        out = memoryview((C.c_uint8 * out_n.value).from_address(p)).cast("B") if out_n.value else memoryview(b"")
        return [(res[i].status, out[res[i].out_off:res[i].out_off + members[i][2]]) for i in range(k)]

    def run_device(self, n, members, tables=None):
        """run() with the decoded members left on the device: [(status, (device address, size))], the addresses
        multiples of 16 inside one buffer and valid until the next run."""
        return self.run(n, members, device=True, tables=tables)

    def stats(self):
        d = dict(self._stats)
        d["kernel_ms"] = sum(d.get(k, 0.0) for k in ("copy_ms", "small_ms", "find_ms", "count_ms", "decode_ms",
                                                      "resolve_ms", "crc_ms"))
        return d

    def close(self):
        if self._u is not None:
            self._ctx.lib.lb2_unzip_destroy(self._u)
            self._u = None
        for attr in ("_in", "_out"):
            if getattr(self, attr) is not None:
                self._ctx.pinned_free(getattr(self, attr))
                setattr(self, attr, None)
                setattr(self, attr + "_cap", 0)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def target_path(zf, member, path):
    """Where ZipFile._extract_member (Python 3.12) puts `member` under `path`, its parent directories made: the name
    with drive letters, absolute roots, "." and ".." dropped."""
    arcname = member.filename.replace("/", os.path.sep)
    if os.path.altsep:
        arcname = arcname.replace(os.path.altsep, os.path.sep)
    arcname = os.path.splitdrive(arcname)[1]
    invalid_path_parts = ("", os.path.curdir, os.path.pardir)
    arcname = os.path.sep.join(x for x in arcname.split(os.path.sep) if x not in invalid_path_parts)
    if os.path.sep == "\\":
        arcname = zf._sanitize_windows_name(arcname, os.path.sep)
    if not arcname and not member.is_dir():
        raise ValueError("Empty filename.")
    targetpath = os.path.normpath(os.path.join(path, arcname))
    upperdirs = os.path.dirname(targetpath)
    if upperdirs and not os.path.exists(upperdirs):
        os.makedirs(upperdirs)
    return targetpath


def _gpu_member(zi):
    return zi.compress_type in _GPU_METHODS and not zi.flag_bits & _STDLIB_FLAGS and not zi.is_dir()


def _body(zf, zi, buf, lo, archive_bytes):
    """(offset of zi's body in buf, its length) after the checks ZipFile.open makes on the local header, or None when
    a check fails (the stdlib's own code then raises what it raises)."""
    off = zi.header_offset - lo
    if off < 0 or off + zipfile.sizeFileHeader > len(buf):
        return None
    fh = struct.unpack(zipfile.structFileHeader, buf[off:off + zipfile.sizeFileHeader])
    if fh[zipfile._FH_SIGNATURE] != zipfile.stringFileHeader:
        return None
    name_end = off + zipfile.sizeFileHeader + fh[zipfile._FH_FILENAME_LENGTH]
    if name_end > len(buf):
        return None
    fname = bytes(buf[off + zipfile.sizeFileHeader:name_end])
    try:
        fname = fname.decode("utf-8" if fh[zipfile._FH_GENERAL_PURPOSE_FLAG_BITS] & 0x800 else
                             (zf.metadata_encoding or "cp437"))
    except UnicodeDecodeError:
        return None
    if fname != zi.orig_filename:
        return None
    body = name_end + fh[zipfile._FH_EXTRA_FIELD_LENGTH]
    end_offset = getattr(zi, "_end_offset", None)
    if end_offset is not None and lo + body + zi.compress_size > end_offset:
        return None
    if lo + body + zi.compress_size > archive_bytes:
        return body, -1  # the file ends inside the body (ZipExtFile raises EOFError)
    return body, zi.compress_size


class _Reader:
    """Decodes the GPU members of a run of entries, batch by batch, with the archive file's bytes read once."""

    def __init__(self, zf, fp, decoder, batch_bytes):
        self.zf, self.fp, self.decoder, self.batch_bytes = zf, fp, decoder, batch_bytes
        fp.seek(0, os.SEEK_END)
        self.archive_bytes = fp.tell()
        self.n_gpu = self.n_stdlib = self.n_batches = 0
        self.in_bytes = self.out_bytes = 0

    def batches(self, entries):
        """yield (entries of one batch, {id(ZipInfo): (status, data)} of its GPU members)"""
        batch, cost = [], 0
        for zi in entries:
            c = zi.compress_size + 3 * zi.file_size + 1024
            if batch and cost + c > self.batch_bytes:
                yield batch, self.decode(batch)
                batch, cost = [], 0
            batch.append(zi)
            cost += c
        if batch:
            yield batch, self.decode(batch)

    def decode(self, batch):
        todo = list({id(zi): zi for zi in batch if _gpu_member(zi)}.values())
        got = {}
        self._decode(todo, got)
        self.n_batches += 1
        return got

    def _decode(self, todo, got):
        if not todo:
            return
        lo = min(zi.header_offset for zi in todo)
        hi = min(self.archive_bytes, max(zi.header_offset + zipfile.sizeFileHeader + 2 * 65535 + zi.compress_size
                                         for zi in todo))
        buf = self.decoder.buffer(max(hi - lo, 0))
        self.fp.seek(lo)
        _read_into(self.fp, buf)
        members, infos, tables = [], [], []
        for zi in todo:
            b = _body(self.zf, zi, buf, lo, self.archive_bytes)
            if b is not None and b[1] < 0:
                got[id(zi)] = (UNZIP_BAD_DATA, None)
            elif b is not None:
                members.append((b[0], b[1], zi.file_size, zi.CRC, zi.compress_type))
                infos.append(zi)
                tables.append(_seek_entries(zi))
        try:
            res = self.decoder.run(len(buf), members, tables=tables) if any(tables) else \
                self.decoder.run(len(buf), members)
        except DeviceTooSmall:
            if len(infos) == 1:
                return  # does not fit on the device alone: the stdlib's code reads it
            half = len(infos) // 2
            self._decode(infos[:half], got)
            self._decode(infos[half:], got)
            return
        for zi, (status, data) in zip(infos, res):
            got[id(zi)] = (status, bytes(data) if status == UNZIP_OK else None)
            self.n_gpu += 1
            self.in_bytes += zi.compress_size
            self.out_bytes += zi.file_size

    def stats(self, n_members):
        st = {"members": n_members, "gpu_members": self.n_gpu, "batches": self.n_batches, "in_bytes": self.in_bytes,
              "out_bytes": self.out_bytes}
        st.update(self.decoder.stats())
        return st


def _seek_entries(zi):
    """the seek table of a DEFLATE member from its central-directory extra field, or None (none, or not valid)"""
    if zi.compress_type != zipfile.ZIP_DEFLATED:
        return None
    entries = ST.zip_entries(zi.extra)
    return entries if ST.valid(entries, zi.compress_size, zi.file_size) else None


def _raise_for(zi, status):
    if status == UNZIP_BAD_CRC:
        raise zipfile.BadZipFile("Bad CRC-32 for file %r" % zi.filename)
    raise BadZipMember(zi.filename, "Invalid DEFLATE data" if status == UNZIP_BAD_DATA else "Wrong uncompressed size")


def extract_with(zip_path, directory, decoder, batch_bytes=BATCH_BYTES):
    """extract_zip with the member bodies decoded by `decoder` (GpuUnzipDecoder, or a stand-in with the same
    interface)."""
    path = os.fspath(directory)
    with zipfile.ZipFile(zip_path) as zf, open(zip_path, "rb") as fp:
        entries = [zf.getinfo(name) for name in zf.namelist()]  # as extractall: a repeated name is its last entry
        r = _Reader(zf, fp, decoder, batch_bytes)
        n_files = n_stdlib = 0
        for batch, got in r.batches(entries):
            for zi in batch:  # the whole batch is checked before any of its files is written
                status = got.get(id(zi), (UNZIP_OK, None))[0]
                if status != UNZIP_OK:
                    _raise_for(zi, status)
            for zi in batch:
                if id(zi) in got:
                    with open(target_path(zf, zi, path), "wb") as f:
                        f.write(got[id(zi)][1])
                    n_files += 1
                else:
                    n_stdlib += not zi.is_dir()
                    zf.extract(zi, path)
    st = r.stats(len(entries))
    st.update(files=n_files, stdlib_members=n_stdlib)
    return st


def testzip_with(zip_path, decoder, batch_bytes=BATCH_BYTES):
    """testzip with the member bodies decoded by `decoder`; returns (name or None, stats)."""
    with zipfile.ZipFile(zip_path) as zf, open(zip_path, "rb") as fp:
        listed = list(zf.filelist)
        byname = {id(zi): zf.getinfo(zi.filename) for zi in listed}  # ZipFile.testzip opens each entry by its name
        r = _Reader(zf, fp, decoder, batch_bytes)
        pos = 0
        n_stdlib = 0
        for batch, got in r.batches([byname[id(zi)] for zi in listed]):
            for zi in batch:
                name = listed[pos].filename
                pos += 1
                if id(zi) in got:
                    if got[id(zi)][0] != UNZIP_OK:
                        return name, r.stats(len(listed))
                    continue
                n_stdlib += not zi.is_dir()
                try:
                    with zf.open(zi, "r") as f:
                        while f.read(1 << 20):
                            pass
                except zipfile.BadZipFile:
                    return name, r.stats(len(listed))
    st = r.stats(len(listed))
    st["stdlib_members"] = n_stdlib
    return None, st


def _with_decoder(ctx, fn):
    from .tarball import _default_context
    own = False
    if ctx is None:
        ctx, own = _default_context()
    try:
        with GpuUnzipDecoder(ctx) as dec:
            return fn(dec)
    finally:
        if own:
            ctx.close()


def extract_zip(zip_path, directory, ctx=None, batch_bytes=BATCH_BYTES):
    """Extract `zip_path` under `directory` as `ZipFile(zip_path).extractall(directory)` does -- the same paths (".."
    components, drive letters and absolute names sanitised as its _extract_member does), directories and contents,
    in archive order -- with every STORED and DEFLATE member decoded and CRC-checked on the GPU.  Members are decoded
    in batches bounded by device memory; a batch is decoded and checked before any of its files is written.

    A CRC mismatch raises zipfile.BadZipFile("Bad CRC-32 for file %r"), as the stdlib does; invalid DEFLATE data or a
    wrong size raises BadZipMember (a BadZipFile) naming the member.  Encrypted members, other methods (bzip2, lzma,
    deflate64), members whose local header the stdlib would refuse and members that do not fit on the device alone
    are extracted by the stdlib's own code.  Returns a stats dict: members, gpu_members, stdlib_members, files,
    batches, in_bytes, out_bytes, kernel_ms and the lb2_unzip_stats fields summed over the batches.  ctx=None: the
    context the strip path has already warmed up, if any, else a new one.  There is no CPU path: without a GPU this
    raises."""
    return _with_decoder(ctx, lambda dec: extract_with(zip_path, directory, dec, batch_bytes))


def testzip(zip_path, ctx=None, batch_bytes=BATCH_BYTES):
    """The name of the first bad member of `zip_path`, or None, as `ZipFile(zip_path).testzip()` returns it, with
    every STORED and DEFLATE member decoded and CRC-checked on the GPU.  One difference: where the stdlib raises
    instead of naming the member -- zlib.error for invalid DEFLATE data, EOFError for a body cut short by its recorded
    sizes -- this returns the member's name.  (A member that decodes to fewer bytes than its recorded size is also
    named; the stdlib passes it when the CRC-32 of the shorter output matches.)"""
    return _with_decoder(ctx, lambda dec: testzip_with(zip_path, dec, batch_bytes)[0])


# ---- strip_zip: inflate, strip and deflate chained on the device -------------------------------------------------
# Three seams, each an object a CPU stand-in can replace: the decoder (`run_device`: members decoded and left in
# device memory), the stripper below and the encoder (`submit_device`: a piece gathered from device memory).  What
# travels between them is a reference, a (device address, length) pair; only those objects look inside one.

SO_SUFFIX = ".so"   # the reference's `find -name "*.so"`
_S_IFMT, _S_IFLNK = 0o170000, 0o120000


class StripFailed(RuntimeError):
    """A selected member that `strip` refuses: where the reference's `xargs strip` exits 123 and the build stops."""

    def __init__(self, name, why):
        super().__init__("%s: %s" % (name, why))
        self.member = name


def host_strip(data):
    """`strip` (the host binary, the reference's own tool) on `data` in a temporary file: the new bytes, or None
    when strip refuses the file."""
    fd, path = tempfile.mkstemp(suffix=SO_SUFFIX)
    try:
        with os.fdopen(fd, "wb") as f:
            f.write(data)
        if subprocess.run(["strip", path], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL).returncode != 0:
            return None
        with open(path, "rb") as f:
            return f.read()
    finally:
        os.unlink(path)


class GpuStripper:
    """lb2_strip_device_async / lb2_batch_results over files that already lie in device memory.

    strip(refs): refs are (address, size) with every address a multiple of 16 (each file is read at its own address,
    so they may lie in several device buffers, such as a tar arena and the decoder's output); returns [(LB2_ST_* status, (address, size) of the stripped file in the output arena)], valid until
    the next strip().  fetch(ref) brings a file to the host and upload(data) puts one on the device (until the next
    strip()): the two directions of the host-strip fallback, counted in uploaded / downloaded.  host_strip is the
    fallback itself."""

    host_strip = staticmethod(host_strip)

    def __init__(self, ctx):
        self._ctx, self._out, self._cap, self._extra = ctx, None, 0, []
        self.uploaded = self.downloaded = 0
        self._stats = {"plan_ms": 0.0, "compact_ms": 0.0}

    def _release(self):
        for p in self._extra:
            self._ctx.dev_free(p)
        self._extra = []

    def strip(self, refs):
        self._release()
        n = len(refs)
        if not n:
            return []
        base = min(a for a, _ in refs)
        off = (C.c_uint64 * (n + 1))(*[a - base for a, _ in refs], 0)
        sizes = (C.c_uint64 * n)(*[k for _, k in refs])
        need = sum(-(-k // 256) * 256 for _, k in refs) + 4096 * n + (1 << 20)
        out_off, out_sizes, status, st = (C.c_uint64 * (n + 1))(), (C.c_uint64 * n)(), (C.c_int32 * n)(), N.Stats()
        lib, ctx = self._ctx.lib, self._ctx
        while True:
            if need > self._cap:
                if self._out is not None:
                    ctx.dev_free(self._out)
                    self._out, self._cap = None, 0
                self._out = ctx.dev_alloc(need)
                self._cap = need
            ctx.check(lib.lb2_strip_device_async(ctx.h, base, off, sizes, n, self._out, self._cap, 0, None))
            rc = lib.lb2_batch_results(ctx.h, out_off, out_sizes, status, C.byref(st))
            if rc == N.LB2_E_CAPACITY and st.out_bytes_needed + (1 << 20) > self._cap:  # re-laid-out files can grow
                need = st.out_bytes_needed + (1 << 20)
                continue
            ctx.check(rc)
            break
        self._stats["plan_ms"] += st.plan_ms
        self._stats["compact_ms"] += st.compact_ms
        return [(status[i], (self._out + out_off[i], out_sizes[i])) for i in range(n)]

    def fetch(self, ref):
        addr, n = ref
        buf = C.create_string_buffer(n)
        if n:
            self._ctx.d2h(buf, addr, n)
        self.downloaded += n
        return buf.raw

    def upload(self, data):
        p = self._ctx.dev_alloc(len(data))
        self._extra.append(p)
        if data:
            self._ctx.h2d(p, data, len(data))
        self.uploaded += len(data)
        return p, len(data)

    def stats(self):
        return dict(self._stats)

    def close(self):
        self._release()
        if self._out is not None:
            self._ctx.dev_free(self._out)
            self._out, self._cap = None, 0

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def selected_for_strip(zi):
    """None: the reference's line never sees the member; True: a regular file `find -name "*.so"` hands to strip;
    False: a matching name that is a directory entry or (by its Unix mode) a symlink, which is left alone."""
    name = zi.filename[:-1] if zi.is_dir() else zi.filename
    if not name.rsplit("/", 1)[-1].endswith(SO_SUFFIX):
        return None
    return not zi.is_dir() and (zi.external_attr >> 16) & _S_IFMT != _S_IFLNK


def _kept(zi):
    """A copy of a source archive's ZipInfo for the archive being written: no data descriptor (the sizes are known),
    no zip64 extra field (FileHeader and central_directory make their own), no seek table (it belongs in the central
    directory only: strip_with hands it to the writer's tables)."""
    out = copy.copy(zi)
    out.flag_bits &= ~zipfile._MASK_USE_DATA_DESCRIPTOR
    out.extra = zipfile._strip_extra(zi.extra, (1, ST.ZIP_ID))
    return out


def _device_pieces(items, piece, max_segs):
    """Cut items [(entry index, (address, size))] into pieces as write_zip cuts files: yields ([(entry index,
    (address, bytes))], flags); a file that does not fit in the rest of a piece leaves a multiple of CHUNK in it."""
    fill, segs, cont = 0, [], False
    for idx, (addr, n) in items:
        pos = 0
        while True:
            off = -(-fill // ALIGN) * ALIGN
            if len(segs) == max_segs or off > piece or (n - pos > piece - off and piece - off < CHUNK):
                yield segs, N.ZIP_CONTINUES if cont else 0
                segs, cont, off = [], False, 0
            want = n - pos if n - pos <= piece - off else (piece - off) // CHUNK * CHUNK
            segs.append((idx, (addr + pos, want)))
            fill, pos = off + want, pos + want
            if pos == n:
                break
            yield segs, (N.ZIP_CONTINUES if cont else 0) | N.ZIP_MORE
            fill, segs, cont = 0, [], True
    if segs:
        yield segs, N.ZIP_CONTINUES if cont else 0


def decode_members(decoder, batch, consume, _whole=True):
    """Inflate the members of a batch [(key, ZipInfo, (ZipFile, its open file, its size))] on the device: every body is
    read into one upload buffer and the decoder's run_device takes them all, reading a member's seek table when it has
    one.  When the batch does not fit on the device (DeviceTooSmall) it is split in halves, each decoded on its own.
    consume(part, decoded, whole) is called once per part that was decoded, in order: part is a slice of the batch,
    decoded {key: (UNZIP_* status, (device address, size))} holds the members the decoder took, valid until the
    decoder's next run (the next part's, when the batch was split), and whole says whether part is the entire batch.
    A member the GPU reader does not take (another method, encryption, a local header the stdlib refuses) or that
    does not fit on the device alone has no entry: the stdlib's own code reads it.  Returns the body bytes uploaded."""
    view = decoder.buffer(sum(zi.compress_size for _, zi, _ in batch))
    members, taken, tables, fill = [], [], [], 0
    for key, zi, (zf, src, archive_bytes) in batch:
        if not _gpu_member(zi):
            continue
        src.seek(zi.header_offset)
        head = src.read(zipfile.sizeFileHeader)
        if len(head) == zipfile.sizeFileHeader:
            fh = struct.unpack(zipfile.structFileHeader, head)
            head += src.read(fh[zipfile._FH_FILENAME_LENGTH] + fh[zipfile._FH_EXTRA_FIELD_LENGTH])
        b = _body(zf, zi, head, zi.header_offset, archive_bytes)
        if b is None or b[0] != len(head):
            continue                       # the stdlib's own code reads it, and raises what it raises
        if b[1] < 0 or _read_into(src, view[fill:fill + zi.compress_size]) != zi.compress_size:
            raise BadZipMember(zi.filename, "The archive ends inside the body")
        members.append((fill, zi.compress_size, zi.file_size, zi.CRC, zi.compress_type))
        taken.append(key)
        tables.append(_seek_entries(zi))
        fill += zi.compress_size
    decoded, uploaded = {}, 0
    try:
        if taken:
            res = decoder.run_device(fill, members, tables=tables) if any(tables) else decoder.run_device(fill, members)
            decoded, uploaded = dict(zip(taken, res)), fill
    except DeviceTooSmall:
        if len(taken) > 1:
            half = len(batch) // 2
            return decode_members(decoder, batch[:half], consume, False) + \
                decode_members(decoder, batch[half:], consume, False)
        # a member that does not fit on the device alone: read by the stdlib
    consume(batch, decoded, _whole)
    return uploaded


def strip_with(src_zip, dst_zip, decoder, stripper, encoder, fallback_host_strip=True, tolerate_non_elf=False,
               batch_bytes=BATCH_BYTES):
    """strip_zip with the three engines given (GpuUnzipDecoder, GpuStripper, GpuZipEncoder, or stand-ins with the
    same interfaces)."""
    src_zip, dst_zip = os.fspath(src_zip), os.fspath(dst_zip)
    if os.path.realpath(src_zip) == os.path.realpath(dst_zip) or \
            (os.path.exists(dst_zip) and os.path.samefile(src_zip, dst_zip)):
        raise ValueError("strip_zip: %r is the archive being read; write the result somewhere else" % dst_zip)
    piece, max_segs = encoder.piece_bytes, encoder.max_segs
    if piece < CHUNK:
        raise ValueError("pieces of %d bytes: at least %d are needed" % (piece, CHUNK))
    out_dir = os.path.dirname(dst_zip) or "."
    os.makedirs(out_dir, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix=os.path.basename(dst_zip) + ".", suffix=".tmp", dir=out_dir)
    try:
        with os.fdopen(fd, "w+b") as fp, zipfile.ZipFile(src_zip) as zf, open(src_zip, "rb") as src:
            src.seek(0, os.SEEK_END)
            archive_bytes = src.tell()
            entries = [(None, _kept(zi)) for zi in zf.filelist]
            n = {"selected": 0, "gpu": 0, "fallback": 0, "skipped": 0, "in_bytes": 0, "uploaded": 0, "downloaded": 0}

            def local_body(zi):
                """the offset of zi's body in src, from its local header"""
                src.seek(zi.header_offset)
                fh = src.read(zipfile.sizeFileHeader)
                if len(fh) != zipfile.sizeFileHeader or fh[:4] != zipfile.stringFileHeader:
                    raise zipfile.BadZipFile("Bad magic number for file header of %r" % zi.filename)
                fh = struct.unpack(zipfile.structFileHeader, fh)
                return zi.header_offset + zipfile.sizeFileHeader + fh[zipfile._FH_FILENAME_LENGTH] + \
                    fh[zipfile._FH_EXTRA_FIELD_LENGTH]

            origin = {id(out): zi for (_, out), zi in zip(entries, zf.filelist)}  # entry written -> the source's

            def copy_member(out):
                zi = origin[id(out)]
                start = local_body(zi)
                fp.write(out.FileHeader())
                src.seek(start)
                left = zi.compress_size
                while left:
                    block = src.read(min(left, 1 << 20))
                    if not block:
                        raise zipfile.BadZipFile("%s ends inside the body of %r" % (src_zip, zi.filename))
                    fp.write(block)
                    left -= len(block)

            w = _ContainerWriter(fp, entries, copy=copy_member)
            source = (zf, src, archive_bytes)
            for idx, zi in enumerate(zf.filelist):   # a member copied as it is keeps its seek table
                field = ST.zip_field_of(zi.extra)
                if field:
                    w.tables[idx] = field
            in_flight = []

            def collect():
                body, res = encoder.collect()
                n["downloaded"] += len(body)
                chunks = getattr(encoder, "seek_chunks", None) or [None] * len(res)
                for (idx, (_, nbytes)), (off, k, crc, ended), ch in zip(in_flight.pop(0), res, chunks):
                    w.part(idx, body[off:off + k], crc, ended, nbytes, ch)

            def host_path(idx, zi, data):
                """the stripped bytes of a member the device did not strip, on the device; None: keep the member"""
                new = stripper.host_strip(data) if fallback_host_strip else None
                if new is None:
                    if tolerate_non_elf and data[:4] != b"\x7fELF":
                        n["skipped"] += 1
                        return None
                    raise StripFailed(zi.filename, "strip refuses this file (the reference's xargs exits 123)"
                                      if fallback_host_strip else "not stripped on the GPU, and the host strip is off")
                n["fallback"] += 1
                return stripper.upload(new)

            def run(batch):
                """batch: [(entry index, source ZipInfo)] of selected members, in archive order"""
                n["uploaded"] += decode_members(decoder, [(idx, zi, source) for idx, zi in batch], finish)

            def finish(part, decoded, whole):
                batch = [(idx, zi) for idx, zi, _ in part]
                for idx, zi in batch:
                    status = decoded.get(idx, (UNZIP_OK, None))[0]
                    if status != UNZIP_OK:
                        raise BadZipMember(zi.filename, {UNZIP_BAD_DATA: "Invalid DEFLATE data", UNZIP_BAD_CRC: "Bad CRC-32",
                                                         UNZIP_WRONG_SIZE: "Wrong uncompressed size"}[status])
                on_device = [(idx, zi) for idx, zi in batch if idx in decoded]
                stripped = dict(zip([idx for idx, _ in on_device],
                                    stripper.strip([decoded[idx][1] for idx, _ in on_device])))
                items = []
                for idx, zi in batch:
                    if idx in stripped and stripped[idx][0] == N.ST_OK:
                        ref = stripped[idx][1]
                        n["gpu"] += 1
                    elif idx in stripped and stripped[idx][0] == N.ST_NOT_ELF and tolerate_non_elf:
                        n["skipped"] += 1
                        continue
                    else:
                        ref = host_path(idx, zi, stripper.fetch(decoded[idx][1]) if idx in decoded else zf.read(zi))
                        if ref is None:
                            continue
                    entries[idx][1].file_size = ref[1]   # the writer's zip64 choice is made from it
                    n["in_bytes"] += zi.file_size
                    items.append((idx, ref))
                for segs, flags in _device_pieces(items, piece, max_segs):
                    encoder.submit_device([ref for _, ref in segs], flags)
                    in_flight.append(segs)
                    if len(in_flight) == 2:
                        collect()
                while in_flight:  # the next batch replaces the buffers these pieces read
                    collect()

            batch, cost = [], 0
            for idx, zi in enumerate(zf.filelist):
                sel = selected_for_strip(zi)
                if not sel:
                    n["skipped"] += sel is False
                    continue
                n["selected"] += 1
                c = zi.compress_size + 4 * zi.file_size + 1024
                if batch and cost + c > batch_bytes:
                    run(batch)
                    batch, cost = [], 0
                batch.append((idx, zi))
                cost += c
            if batch:
                run(batch)
            w.finish(zf.comment)
            zip_bytes = fp.tell()
        os.chmod(tmp, 0o666 & ~_umask())
        os.replace(tmp, dst_zip)
    except BaseException:
        os.unlink(tmp)
        raise
    st = {"members": len(entries), "selected": n["selected"], "gpu": n["gpu"], "fallback": n["fallback"],
          "skipped": n["skipped"], "in_bytes": n["in_bytes"], "out_bytes": w.in_bytes, "deflated_bytes": w.out_bytes,
          "src_zip_bytes": archive_bytes, "zip_bytes": zip_bytes,
          "uploaded_bytes": n["uploaded"] + stripper.uploaded, "downloaded_bytes": n["downloaded"] + stripper.downloaded,
          "unzip": decoder.stats(), "strip": stripper.stats(), "deflate": encoder.stats()}
    st["kernel_ms"] = st["unzip"].get("kernel_ms", 0.0) + sum(st["strip"].values()) + st["deflate"].get("kernel_ms", 0.0)
    return st


def _umask():
    mask = os.umask(0)
    os.umask(mask)
    return mask


def strip_zip(src_zip, dst_zip, ctx=None, compresslevel=None, fallback_host_strip=True, tolerate_non_elf=False,
              batch_bytes=BATCH_BYTES, piece_bytes=PIECE_BYTES, seek_table=False):
    """Write `dst_zip` with the members of `src_zip`, in their order, every `*.so` member stripped: the archive that
    `ZipFile(src_zip).extractall(d)`, the reference's `find d/ -name "*.so" | xargs strip` and a zip of `d` lead to,
    without the tree.  src_zip is only read; dst_zip appears under its name when it is complete, and not at all when
    the call raises; dst_zip == src_zip raises ValueError.

    Selected: regular-file members whose basename ends in ".so" (directory entries and members whose Unix mode says
    symlink are counted as skipped).  In batches bounded by device memory their bodies are uploaded, inflated and
    CRC-checked (lb2_unzip_run), stripped where they lie (lb2_strip_device_async) and deflated from the stripped arena
    (lb2_zip_submit_device), so only compressed bytes cross the bus; each becomes a ZIP_DEFLATED member with its new
    CRC-32 and sizes.  Every other member's body, method, CRC-32, sizes, name, time, attributes, extra field and
    comment are copied as they are under a fresh local header (no data descriptor; zip64 fields regenerated); the
    archive comment is kept, bytes in front of the first member are not.

    An ELF the planner refuses is fetched, stripped by the host `strip` and uploaded again (fallback_host_strip), as
    in strip_tree; so is a selected member the GPU reader does not take (encrypted, bzip2 ...: the stdlib reads it
    and raises what it raises).  A member `strip` refuses raises StripFailed -- the reference's xargs exits 123 --
    unless it is not an ELF and tolerate_non_elf keeps it as it is.  A member that does not read back raises
    BadZipMember.  compresslevel: None or 9, as zip_tree.  A source member's seek table is used to read it; a member
    copied as it is keeps its table in the central directory, a rewritten one drops it and, with seek_table=True,
    gets a new one, as zip_tree writes it.

    Returns a stats dict: members, selected, gpu, fallback, skipped; in_bytes / out_bytes (the stripped members
    before and after) and deflated_bytes (their new bodies); src_zip_bytes, zip_bytes; uploaded_bytes,
    downloaded_bytes (everything that crossed the bus for member data); unzip, strip (plan_ms, compact_ms) and
    deflate (the three engines' stats) and kernel_ms, their kernel times summed.  There is no CPU path: without a
    GPU this raises."""
    from .tarball import _default_context
    N.deflate_flags(compresslevel)
    own = False
    if ctx is None:
        ctx, own = _default_context()
    try:
        with GpuUnzipDecoder(ctx) as dec, GpuStripper(ctx) as stripper, \
                GpuZipEncoder(ctx, piece_bytes, compresslevel=compresslevel, host_buffers=False, seek_table=seek_table) as enc:
            return strip_with(src_zip, dst_zip, dec, stripper, enc, fallback_host_strip, tolerate_non_elf, batch_bytes)
    finally:
        if own:
            ctx.close()


def main(argv=None):
    """python -m lambdipy_b200.zipfile_gpu strip SRC DST [--level 9] [--seek-table]"""
    import argparse
    from . import patch, project_build
    ap = argparse.ArgumentParser(prog="python -m lambdipy_b200.zipfile_gpu")
    sub = ap.add_subparsers(dest="command", required=True)
    sp = sub.add_parser("strip", help="strip the *.so members of SRC on the GPU and write the result to DST")
    sp.add_argument("src")
    sp.add_argument("dst")
    sp.add_argument("--level", type=int, choices=[9], default=None, help="9: the optimal parse (smaller, slower)")
    sp.add_argument("--seek-table", action="store_true",
                    help="give the rewritten members seek tables, with which the GPU reader decodes them without search")
    args = ap.parse_args(argv)
    st = strip_zip(args.src, args.dst, compresslevel=args.level, **seek_kw(args.seek_table))
    with zipfile.ZipFile(args.dst) as zf:
        unzipped = sum(zi.file_size for zi in zf.filelist)
    print("Bundle zip: %s, %.1f MB = %.0f %% of the 50 MB direct-upload limit; unzipped %.1f MB = %.0f %% of 250 MB; "
          "%d shared objects stripped (%d via host strip), %.1f MB -> %.1f MB"
          % (args.dst, st["zip_bytes"] / 1e6, 100.0 * st["zip_bytes"] / patch.LAMBDA_ZIPPED_LIMIT, unzipped / 1e6,
             100.0 * unzipped / project_build.LAMBDA_UNZIPPED_LIMIT, st["gpu"] + st["fallback"], st["fallback"],
             st["in_bytes"] / 1e6, st["out_bytes"] / 1e6))
    return 0


if __name__ == "__main__":
    sys.exit(main())
