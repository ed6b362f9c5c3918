"""Raw-DEFLATE streams for the inflate tests: zlib's levels, memLevel extremes, strategies and flush modes over text,
real shared-object bytes, random bytes and zeros.  Each entry is (name, raw DEFLATE body, decompressed bytes)."""
import glob
import os
import random
import zlib

import numpy as np


def text(n, seed=1):
    rng = random.Random(seed)
    words = ["package", "build", "lambda", "layer", "strip", "tarball", "numpy", "scipy", "the", "of", "and", "a",
             "shared", "object", "section", "symbol", "gzip", "inflate", "block", "window", "\n", "def", "return"]
    out, size = [], 0
    while size < n:
        w = rng.choice(words) + (" " if rng.random() < 0.9 else ",\n")
        out.append(w)
        size += len(w)
    return "".join(out).encode()[:n]


def so_bytes(n):
    """n bytes of real shared objects from numpy's and scipy's trees"""
    site = os.path.dirname(os.path.dirname(np.__file__))
    paths = sorted(glob.glob(os.path.join(site, "numpy*", "**", "*.so*"), recursive=True))
    paths += sorted(glob.glob(os.path.join(site, "scipy*", "**", "*.so*"), recursive=True))
    out = bytearray()
    for p in paths:
        if len(out) >= n:
            break
        if os.path.isfile(p):
            with open(p, "rb") as f:
                out += f.read(n - len(out))
    return bytes(out)


def deflate(data, level=6, mem=8, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=(), seed=0):
    """raw DEFLATE of data; flushes: zlib flush modes issued at random offsets"""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, mem, strategy)
    rng = random.Random(seed)
    cuts = sorted(rng.randrange(1, len(data)) for _ in range(12)) if flushes and len(data) > 1 else []
    out, pos = [], 0
    for k, cut in enumerate(cuts):
        out.append(c.compress(data[pos:cut]))
        out.append(c.flush(flushes[k % len(flushes)]))
        pos = cut
    out.append(c.compress(data[pos:]))
    out.append(c.flush())
    return b"".join(out)


def matrix(size=1 << 20):
    """(name, raw body, data) over the stream matrix, each input about `size` bytes"""
    rnd = random.Random(7).randbytes(size)
    sources = {"text": text(size), "so": so_bytes(size), "random": rnd,
               "mixed": text(size // 4) + rnd[:size // 4] + bytes(size // 4) + so_bytes(size // 4)}
    out = []
    for sname, data in sources.items():
        for level in (0, 1, 6, 9):
            out.append(("%s-l%d" % (sname, level), deflate(data, level), data))
        for mem in (1, 9):
            out.append(("%s-mem%d" % (sname, mem), deflate(data, 9, mem), data))
        for st, sn in ((zlib.Z_FILTERED, "filtered"), (zlib.Z_HUFFMAN_ONLY, "huffman"), (zlib.Z_RLE, "rle"),
                       (zlib.Z_FIXED, "fixed")):
            out.append(("%s-%s" % (sname, sn), deflate(data, 6, 8, st), data))
        for fl, fn in ((zlib.Z_SYNC_FLUSH, "sync"), (zlib.Z_FULL_FLUSH, "full"), (zlib.Z_PARTIAL_FLUSH, "partial")):
            out.append(("%s-%sflush" % (sname, fn), deflate(data, 6, flushes=(fl,), seed=len(out)), data))
    for n in (0, 1, 2, 1023, 1024, 1025, 4095, 4096, 4097):
        data = text(n, seed=n)
        out.append(("edge-%d" % n, deflate(data, 9), data))
    return out
