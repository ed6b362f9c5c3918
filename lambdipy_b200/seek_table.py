"""The seek table: where the DEFLATE blocks of a GPU-written gzip file start, kept in the file itself.

The GPU writers cut a stream into 64 KB chunks and end each one byte-aligned with an empty stored block, so every
chunk starts a block at a known byte.  A seek table records, for each run of consecutive whole chunks, its compressed
and its decoded length.  A reader that trusts nothing but checks everything (lb2_inflate_run_table) then decodes each
run once, from its known start into its known output range, instead of searching for block starts.

This module owns the byte layout; nothing else knows it.

Entries.  A table is a list of (compressed bytes, decoded bytes) entries in stream order, each a pair of unsigned
LEB128 varints.  By default there is one entry per chunk; when that does not fit the field, runs of the smallest k
chunks that fit, a run also ending at a short chunk (the last chunk of a piece).  The last entry's compressed bytes
include the final block (03 00).  A table is written only for two or more entries.

gzip.  The table is one extra gzip member after the unchanged data member:

    1f 8b 08 04 00000000 00 ff  XLEN          header, FLG = FEXTRA only
    'L' 'S' LEN <entries>                       the table
    'L' 'O' 08 00 <u64 LE>                      the file offset of this member's first byte (always last)
    03 00  00000000  00000000                   an empty DEFLATE body, CRC-32 0, ISIZE 0

so an indexed file always ends in the same 22 bytes and a reader finds the table from the tail without decoding
anything.  `gzip`, `tar` and `tarfile` read the file as the data member followed by an empty one, which decompresses
to the same bytes; the file without its last member is byte for byte the file written without a table.

zip.  A DEFLATE member's table is an extra field with header ID ZIP_ID (0x4C53, not in APPNOTE 4.6's list of
assigned IDs) in its central-directory entry only, after the member's other extra fields; the local headers are
unchanged, so the archive is the no-table archive up to the central directory.  The field holds the entries and is
limited to what the 65 535 bytes of the extra field leave.
"""
import struct

CHUNK = 64 << 10                      # the writers' chunk (GZ_CHUNK)
MAX_RATIO = 1032                      # decoded bytes per compressed byte DEFLATE can reach (258 per 2 bits)
GZIP_HEAD = bytes([0x1F, 0x8B, 8, 4, 0, 0, 0, 0, 0, 0xFF])
GZIP_LIMIT = 0xFFFF - 4 - 12          # XLEN's room for the entries: their subfield header and the offset subfield
TAIL = 22                             # 'L' 'O' 08 00 <u64> 03 00 <CRC-32 0> <ISIZE 0>
ZIP_ID = 0x4C53                       # the zip extra field's header ID


def _varint(v, out):
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return


def encode(entries):
    """the entries as LEB128 varint pairs"""
    out = bytearray()
    for c, u in entries:
        _varint(c, out)
        _varint(u, out)
    return bytes(out)


def decode(data):
    """[(compressed, decoded)] from encode()'s bytes, or None for a truncated varint, an odd count or a value past 64
    bits"""
    vals, v, shift = [], 0, 0
    for b in bytes(data):
        if shift > 63 or (shift == 63 and b & 0x7E):
            return None
        v |= (b & 0x7F) << shift
        if b & 0x80:
            shift += 7
        else:
            vals.append(v)
            v, shift = 0, 0
    if shift or len(vals) % 2:
        return None
    return list(zip(vals[0::2], vals[1::2]))


def runs(chunks, k):
    """chunks [(compressed, decoded)] in stream order grouped into entries of k chunks; a run also ends at a chunk
    shorter than CHUNK (the last one of a piece)"""
    out, c, u, n = [], 0, 0, 0
    for cc, uu in chunks:
        c, u, n = c + cc, u + uu, n + 1
        if n == k or uu < CHUNK:
            out.append((c, u))
            c, u, n = 0, 0, 0
    if n:
        out.append((c, u))
    return out


def build(chunks, limit=GZIP_LIMIT):
    """The entries of a table for `chunks` whose encoding fits `limit` bytes, with the fewest chunks per run that
    fits; None when that gives fewer than two entries (no table is written)."""
    k = 1
    while True:
        entries = runs(chunks, k)
        if len(entries) < 2:
            return None
        if len(encode(entries)) <= limit:
            return entries
        k += 1


def valid(entries, in_len, out_len, out_mask=(1 << 64) - 1):
    """The checks a reader makes before it uses a table: two or more entries, none 0, at most MAX_RATIO decoded bytes
    per compressed byte, compressed bytes summing to in_len and decoded bytes to out_len (compared under out_mask:
    gzip's ISIZE holds the length mod 2^32)."""
    if entries is None or len(entries) < 2:
        return False
    if any(c <= 0 or u <= 0 or u > MAX_RATIO * c for c, u in entries):
        return False
    return sum(c for c, _ in entries) == in_len and sum(u for _, u in entries) & out_mask == out_len & out_mask


def gzip_member(entries, offset):
    """the table member of a gzip file, written at file offset `offset`"""
    table = encode(entries)
    if len(table) > GZIP_LIMIT:
        raise ValueError("a seek table of %d bytes does not fit the gzip extra field" % len(table))
    extra = b"LS" + struct.pack("<H", len(table)) + table + b"LO" + struct.pack("<HQ", 8, offset)
    return GZIP_HEAD + struct.pack("<H", len(extra)) + extra + b"\x03\x00" + bytes(8)


def gzip_tail(buf):
    """(offset of the table member, entries) when the file `buf` ends in a well-formed table member, else None.  Only
    the member's own bytes are checked here; whether the entries describe the data member in front of it is valid()'s
    question."""
    n = len(buf)
    if n < TAIL + 16:
        return None
    tail = bytes(buf[n - TAIL:])
    if tail[:4] != b"LO\x08\x00" or tail[12:] != b"\x03\x00" + bytes(8):
        return None
    off = struct.unpack_from("<Q", tail, 4)[0]
    if off > n - TAIL - 16:
        return None
    head = bytes(buf[off:off + 16])
    xlen, ls, tlen = struct.unpack_from("<H2sH", head, 10)
    if head[:10] != GZIP_HEAD or ls != b"LS" or xlen != n - off - 22 or tlen != xlen - 16:
        return None
    entries = decode(buf[off + 16:off + 16 + tlen])
    return None if entries is None else (off, entries)


def zip_field(chunks, other_extra):
    """The central-directory extra field for a zip member of `chunks`, which already has `other_extra` bytes of extra
    fields there; b"" when no table is written."""
    entries = build(chunks, 0xFFFF - other_extra - 4)
    if entries is None:
        return b""
    table = encode(entries)
    return struct.pack("<HH", ZIP_ID, len(table)) + table


def zip_field_of(extra):
    """The whole ZIP_ID field (header included) inside a member's extra fields; empty bytes when there is none"""
    extra, pos = bytes(extra), 0
    while pos + 4 <= len(extra):
        tp, ln = struct.unpack_from("<HH", extra, pos)
        if tp == ZIP_ID:
            return extra[pos:pos + 4 + ln]
        pos += 4 + ln
    return b""


def zip_entries(extra):
    """The entries of the ZIP_ID field in a member's extra fields, or None (no field, or a malformed one)"""
    field = zip_field_of(extra)
    if len(field) < 4 or len(field) != 4 + struct.unpack_from("<H", field, 2)[0]:
        return None
    return decode(field[4:])


def seek_kw(on):
    """the keyword arguments that ask a writer for a seek table: none when `on` is false, so that a call without a
    table is the call made before tables existed"""
    return {"seek_table": True} if on else {}
