"""Raw-DEFLATE streams with seek tables for the seek-table tests: zlib flushed at chunk boundaries, so that every
chunk ends byte-aligned and the next one starts a block at a known byte, and the tables' tampered variants.
Each stream is (name, raw body, decompressed bytes, [(compressed, decoded)] entries)."""
import random
import zlib

import inflate_streams as IS

CHUNK = 64 << 10


def flushed(data, cuts, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flush=zlib.Z_SYNC_FLUSH):
    """data deflated with `flush` after each chunk data[cuts[i]:cuts[i + 1]]; the last chunk ends with Z_FINISH"""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    out, entries = [], []
    bounds = [0] + list(cuts) + [len(data)]
    for i in range(len(bounds) - 1):
        part = data[bounds[i]:bounds[i + 1]]
        b = c.compress(part) + c.flush(flush if i + 2 < len(bounds) else zlib.Z_FINISH)
        out.append(b)
        entries.append((len(b), len(part)))
    return b"".join(out), entries


def every(n, step):
    return list(range(step, n, step))


def matrix(size=1 << 20):
    rnd = random.Random(11).randbytes(size)
    text, so = IS.text(size), IS.so_bytes(size)
    odd = sorted(random.Random(5).sample(range(1, size), 9))
    out = []
    for level in (1, 6, 9):
        out.append(("sync64k-l%d" % level, text, every(size, CHUNK), dict(level=level)))
    out.append(("so-sync64k", so, every(size, CHUNK), {}))
    out.append(("sync-odd", so, odd, {}))
    out.append(("full64k", text, every(size, CHUNK), dict(flush=zlib.Z_FULL_FLUSH)))
    out.append(("fixed64k", text, every(size, CHUNK), dict(strategy=zlib.Z_FIXED)))
    out.append(("stored-random", rnd, every(size, CHUNK), dict(level=0)))
    out.append(("random-l6", rnd, every(size, CHUNK), {}))
    out.append(("fixed-odd", so, odd, dict(strategy=zlib.Z_FIXED)))
    streams = []
    for name, data, cuts, kw in out:
        body, entries = flushed(data, cuts, **kw)
        streams.append((name, body, data, entries))
    return streams


def tampered(entries):
    """[(name, entries)] that no honest table has; each keeps the entry count and, where it can, both sums"""
    e = list(entries)
    assert len(e) >= 3
    out = []

    def moved(i, dc=0, du=0):
        t = list(e)
        t[i] = (t[i][0] + dc, t[i][1] + du)
        t[i + 1] = (t[i + 1][0] - dc, t[i + 1][1] - du)
        return t
    out.append(("start+1byte", moved(0, dc=1)))
    out.append(("start-1byte", moved(1, dc=-1)))
    out.append(("swapped", [e[1], e[0]] + e[2:]))
    out.append(("swapped-in", [(e[1][0], e[0][1]), (e[0][0], e[1][1])] + e[2:]))
    out.append(("inside-block", moved(0, dc=-(e[0][0] // 2))))
    out.append(("wrong-out", moved(1, du=1)))
    out.append(("wrong-out-down", moved(0, du=-1)))
    out.append(("final-early", e[:-1]))                          # the table ends before the final block
    out.append(("sum-over", e[:-1] + [(e[-1][0] + (1 << 30), e[-1][1])]))
    out.append(("zero", [(0, 0)] + e))
    out.append(("oversize", e[:-1] + [(e[-1][0], 1033 * e[-1][0])]))
    out.append(("merged-wrong", [(e[0][0] + e[1][0], e[0][1])] + e[2:]))
    return out
