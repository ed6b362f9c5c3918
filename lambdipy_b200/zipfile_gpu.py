"""Lambda deployment zips with every member's DEFLATE body compressed on the GPU.

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
"""
import ctypes as C
import os
import struct
import zipfile

from . import _native as N

PIECE_BYTES = 64 << 20  # file bytes (and padding) per GPU submission
MAX_SEGS = 1 << 16      # files per piece
ALIGN = 16              # each file starts at a 16-byte-aligned offset of its piece (the CRC kernel's vector loads)
CHUNK = 65536           # the encoder's chunk (GZ_CHUNK): a file continued in the next piece is cut at a multiple of it


class GpuZipEncoder:
    """The lb2_zip_* writer with its two pinned piece buffers.

    buffers[k]: writable memoryview of piece_bytes; submit(k, n, seg_off, seg_len, flags) hands buffers[k][:n] to the
    GPU (flags: N.ZIP_CONTINUES / N.ZIP_MORE); collect() waits for the oldest piece and returns (its DEFLATE bytes,
    [(out_off, out_len, crc32, ended) per segment]); the bytes stay valid until the next collect()."""

    def __init__(self, ctx, piece_bytes=PIECE_BYTES, max_segs=MAX_SEGS):
        self._ctx, self._z, self._ptrs, self._out = ctx, None, [], None
        self.piece_bytes, self.max_segs = int(piece_bytes), int(max_segs)
        try:
            z = C.c_void_p()
            ctx.check(ctx.lib.lb2_zip_create(ctx.h, 0, C.byref(z)))
            self._z = z
            self.buffers = []
            for _ in range(2):
                p = ctx.pinned_alloc(self.piece_bytes)
                self._ptrs.append(p)
                self.buffers.append(memoryview((C.c_uint8 * self.piece_bytes).from_address(p)).cast("B"))
            self._cap = N.zip_bound(self.piece_bytes, self.max_segs)
            self._out = ctx.pinned_alloc(self._cap)
        except BaseException:
            self.close()
            raise
        self._pending = []  # segment count of each piece in flight
        self._stats = N.GzipStats()

    def submit(self, k, n, seg_off, seg_len, flags):
        ns = len(seg_off)
        offs, lens = (C.c_uint64 * ns)(*seg_off), (C.c_uint64 * ns)(*seg_len)
        self._ctx.check(self._ctx.lib.lb2_zip_submit(self._z, self._ptrs[k], n, offs, lens, ns, flags))
        self._pending.append(ns)

    def collect(self):
        ns = self._pending.pop(0)
        segs, n = (N.ZipSegment * ns)(), C.c_uint64()
        self._ctx.check(self._ctx.lib.lb2_zip_collect(self._z, self._out, self._cap, C.byref(n), segs, C.byref(self._stats)))
        body = memoryview((C.c_uint8 * n.value).from_address(self._out)).cast("B") if n.value else memoryview(b"")
        return body, [(s.out_off, s.out_len, s.crc32, bool(s.ended)) for s in segs]

    def stats(self):
        st = self._stats
        return {"kernel_ms": st.deflate_ms + st.crc_ms, "deflate_ms": st.deflate_ms, "crc_ms": st.crc_ms,
                "h2d_ms": st.h2d_ms, "d2h_ms": st.d2h_ms, "n_chunks": st.n_chunks,
                "n_stored_chunks": st.n_stored_chunks, "n_fixed_chunks": st.n_fixed_chunks}

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


def central_directory(infos, start):
    """The central directory of `infos` (written from offset `start`) and the end records, as ZipFile.close() writes
    them: zip64 extras for sizes or offsets beyond ZIP64_LIMIT, zip64 end records beyond 65 535 entries or 4 GiB."""
    out = []
    for zi in infos:
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
    return cd + struct.pack(zipfile.structEndArchive, zipfile.stringEndArchive, 0, 0, count, count, size, offset, 0)


class _ContainerWriter:
    """Writes the entries in order as their bodies arrive: a directory as soon as every entry before it is written;
    a file's local header when its first body bytes arrive, rewritten with the CRC and sizes once it ends (seeking
    back, as ZipFile does on a seekable file)."""

    def __init__(self, fp, entries):
        self.fp, self.entries, self.next = fp, entries, 0
        self.cur = None  # (ZipInfo, zip64) of the file being written
        self.in_bytes = self.out_bytes = self.n_files = 0

    def _upto(self, idx):
        while self.next < idx:
            zi = self.entries[self.next][1]
            assert zi.is_dir(), "file entry %s written out of order" % zi.filename
            zi.compress_size = zi.CRC = 0
            zi.header_offset = self.fp.tell()
            self.fp.write(zi.FileHeader(False))
            self.next += 1

    def part(self, idx, body, crc, ended, file_bytes):
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
        self.fp.write(body)
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
            self.cur = None
            self.next = idx + 1

    def finish(self):
        self._upto(len(self.entries))
        start = self.fp.tell()
        self.fp.write(central_directory([zi for _, zi in self.entries], start))


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
            for (idx, nbytes), (off, n, crc, ended) in zip(in_flight.pop(0), res):
                w.part(idx, body[off:off + n], crc, ended, nbytes)

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


def zip_tree(root_dir, zip_path, ctx=None, piece_bytes=PIECE_BYTES):
    """Write `zip_path` as `shutil.make_archive(zip_path[:-4], "zip", root_dir)` would, with every member's DEFLATE
    body and CRC-32 computed on the GPU.  Returns a stats dict: files, entries, in_bytes (file bytes), out_bytes
    (member bodies), zip_bytes, kernel_ms (deflate + CRC-32 kernels, CUDA events), n_chunks, n_stored_chunks,
    n_fixed_chunks and the copy times.  ctx=None: the context the strip path has already warmed up, if any, else a
    new one on device LAMBDIPY_B200_DEVICE (default 0).  There is no CPU path: without a GPU this raises."""
    from .tarball import _default_context
    own = False
    if ctx is None:
        ctx, own = _default_context()
    try:
        with GpuZipEncoder(ctx, piece_bytes) as enc:
            return write_zip(root_dir, zip_path, enc)
    finally:
        if own:
            ctx.close()
