"""A plain-Python DEFLATE (RFC 1951) reference for the gzip writer and reader tests.  It imports nothing from the
package.

* BitWriter and the block builders (stored, fixed, dynamic) craft streams bit by bit, including streams zlib never
  writes: distances up to 32 768, length 258 as code 284 + 31, one-code and empty distance trees, code-length repeats
  across the HLIT / HDIST boundary, padding in front of a stored block's LEN.  Invalid variants are built with the same
  functions (explicit code lengths, raw symbols, header fields).
* parse(body) decodes a raw DEFLATE body in the style of puff and returns the output and every block's structure.  It
  accepts and refuses exactly what zlib's inflate does; code_ok restates inflate_table's rules.
"""
import heapq

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
         6145, 8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_L = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8   # all 288, as RFC 1951 3.2.6 defines the code
FIXED_D = [5] * 32


class DeflateError(Exception):
    pass


def len_sym(length):
    """3..258 -> (symbol, extra value); 258 is symbol 285"""
    if length == 258:
        return 285, 0
    for i in range(27, -1, -1):
        if LBASE[i] <= length:
            return 257 + i, length - LBASE[i]


def dist_sym(dist):
    """1..32768 -> (symbol, extra value)"""
    for i in range(29, -1, -1):
        if DBASE[i] <= dist:
            return i, dist - DBASE[i]


def canonical(lengths):
    """RFC 1951 3.2.2 codes (MSB-first values) for a list of lengths; symbols of length 0 get None.  Over-subscribed
    lengths still get codes (some collide), so invalid streams can be written with them."""
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for l in lengths:
        if l:
            out.append(nxt[l] & ((1 << l) - 1))
            nxt[l] += 1
        else:
            out.append(None)
    return out


def kraft(lengths):
    """sum of 2^-len over the non-zero lengths, as a multiple of 2^-15"""
    return sum(1 << (15 - l) for l in lengths if l)


def code_ok(lengths, kind):
    """zlib's inflate_table rules (kind 'codes', 'lens' or 'dists'): never over-subscribed; incomplete only for a
    literal/length or distance code whose one code has length 1; no codes at all only for distances (zlib builds an
    all-invalid code-length table then, every length decodes as 0 and the header fails for a missing end-of-block)."""
    nz = [l for l in lengths if l]
    if not nz:
        return kind == "dists"
    k = kraft(nz)
    if k > 1 << 15:
        return False
    if k < 1 << 15:
        return kind != "codes" and max(nz) == 1
    return True


# ---------------------------------------------------------------------------------------------------- writing
class BitWriter:
    """LSB-first bit packer"""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    @property
    def bit(self):
        return len(self.out) * 8 + self.n

    def bits(self, v, n):
        assert 0 <= v < (1 << n) or n == 0 and v == 0, (v, n)
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def huff(self, code, n):
        """a Huffman code, given MSB first (RFC 1951 3.1.1)"""
        self.bits(_rev(code, n), n)

    def align(self, pad=0):
        """pad to a byte boundary with the low bits of `pad`"""
        k = (8 - self.n) & 7
        self.bits(pad & ((1 << k) - 1), k)

    def raw(self, data):
        assert self.n == 0
        self.out += data

    def getvalue(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


class Raw:
    """a literal/length symbol written as given: extra bits `lx`, then (unless dsym is None) a distance symbol with
    extra bits `dx`.  Used for 284 + 31 and for the symbols zlib refuses (286, 287, 30, 31)."""

    def __init__(self, lsym, lx=0, dsym=None, dx=0):
        self.lsym, self.lx, self.dsym, self.dx = lsym, lx, dsym, dx

    def out_len(self):
        if self.lsym < 256:
            return 1
        if 257 <= self.lsym <= 285:
            return LBASE[self.lsym - 257] + self.lx
        return 0


def token_symbols(t):
    """token -> (literal/length symbol, extra value, extra bits, distance symbol or None, extra value, extra bits).
    Tokens: an int is a literal byte, (length, dist) a match, Raw(...) explicit symbols."""
    if isinstance(t, int):
        return t, 0, 0, None, 0, 0
    if isinstance(t, Raw):
        lb = LEXT[t.lsym - 257] if 257 <= t.lsym <= 285 else 0
        db = DEXT[t.dsym] if t.dsym is not None and t.dsym < 30 else 0
        return t.lsym, t.lx, lb, t.dsym, t.dx, db
    length, dist = t
    ls, lx = len_sym(length)
    ds, dx = dist_sym(dist)
    return ls, lx, LEXT[ls - 257], ds, dx, DEXT[ds]


def token_len(t):
    return 1 if isinstance(t, int) else t.out_len() if isinstance(t, Raw) else t[0]


def _rev(code, n):
    return int(format(code, "0%db" % n)[::-1], 2) if n else 0


def write_tokens(w, tokens, lcode, llen, dcode, dlen, eob=True):
    lr = [_rev(c, l) for c, l in zip(lcode, llen)]
    dr = [_rev(c, l) for c, l in zip(dcode, dlen)]
    for t in tokens:
        if isinstance(t, int):
            w.bits(lr[t], llen[t])
            continue
        ls, lx, lb, ds, dx, db = token_symbols(t)
        w.bits(lr[ls], llen[ls])
        w.bits(lx, lb)
        if ds is not None:
            w.bits(dr[ds], dlen[ds])
            w.bits(dx, db)
    if eob:
        w.bits(lr[256], llen[256])


def huffman_lengths(freqs):
    """optimal (unconstrained) Huffman code lengths by heapq; a single used symbol gets length 1"""
    items = [(f, i, None) for i, f in enumerate(freqs) if f]
    out = [0] * len(freqs)
    if len(items) == 1:
        out[items[0][1]] = 1
        return out
    heap = [(f, k, [i]) for k, (f, i, _) in enumerate(items)]
    heapq.heapify(heap)
    k = len(heap)
    while len(heap) > 1:
        fa, _, a = heapq.heappop(heap)
        fb, _, b = heapq.heappop(heap)
        for s in a + b:
            out[s] += 1
        heapq.heappush(heap, (fa + fb, k, a + b))
        k += 1
    return out


def limited_lengths(freqs, maxbits):
    """optimal code lengths of at most maxbits (package-merge); a single used symbol gets length 1"""
    used = sorted((f, i) for i, f in enumerate(freqs) if f)
    out = [0] * len(freqs)
    if len(used) == 1:
        out[used[0][1]] = 1
        return out
    leaves = [(f, [i]) for f, i in used]
    pk = list(leaves)
    for _ in range(maxbits - 1):
        merged = [(pk[j][0] + pk[j + 1][0], pk[j][1] + pk[j + 1][1]) for j in range(0, len(pk) - 1, 2)]
        pk = sorted(leaves + merged, key=lambda x: x[0])
    for _, syms in pk[:2 * len(used) - 2]:
        for s in syms:
            out[s] += 1
    return out


def code_cost(freqs, lengths):
    return sum(f * l for f, l in zip(freqs, lengths))


def rle_lengths(lens, allowed=range(19)):
    """code-length symbols (sym, extra) for a length sequence, runs crossing the HLIT / HDIST boundary; 16 / 17 / 18
    only when in `allowed`"""
    out, i = [], 0
    while i < len(lens):
        v, run = lens[i], 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while run >= 11 and 18 in allowed:
                r = min(run, 138)
                out.append((18, r - 11))
                run -= r
            while run >= 3 and 17 in allowed:
                r = min(run, 10)
                out.append((17, r - 3))
                run -= r
        else:
            out.append((v, 0))
            run -= 1
            while run >= 3 and 16 in allowed:
                r = min(run, 6)
                out.append((16, r - 3))
                run -= r
        out += [(v, 0)] * run
    return out


def token_freqs(tokens, eob=True):
    lf, df = [0] * 288, [0] * 32
    for t in tokens:
        ls, _, _, ds, _, _ = token_symbols(t)
        lf[ls] += 1
        if ds is not None:
            df[ds] += 1
    if eob:
        lf[256] += 1
    return lf, df


_FIXED_CODES = (canonical(FIXED_L), canonical(FIXED_D))


class Stream:
    """A raw DEFLATE body under construction; `nout` counts the output bytes written so far."""

    def __init__(self):
        self.w = BitWriter()
        self.nout = 0

    @property
    def bit(self):
        return self.w.bit

    def body(self):
        return self.w.getvalue()

    def stored(self, data, final=False, pad=0, length=None, nlength=None):
        """a stored block; pad: value of the padding bits between the header and LEN (zlib ignores them)"""
        w = self.w
        w.bits(1 if final else 0, 1)
        w.bits(0, 2)
        w.align(pad)
        n = len(data) if length is None else length
        w.bits(n, 16)
        w.bits((~n & 0xFFFF) if nlength is None else nlength, 16)
        w.raw(data)
        self.nout += len(data)

    def fixed(self, tokens, final=False, eob=True):
        w = self.w
        w.bits(1 if final else 0, 1)
        w.bits(1, 2)
        write_tokens(w, tokens, _FIXED_CODES[0], FIXED_L, _FIXED_CODES[1], FIXED_D, eob)
        self.nout += sum(token_len(t) for t in tokens)

    def dynamic(self, tokens, final=False, llens=None, dlens=None, cl_lens=None, rle=None, hlit=None, hdist=None,
                hclen=None, eob=True):
        """A dynamic block.  Defaults: optimal 15-bit codes for the tokens (two distance codes at least unless
        `dlens` is given), the code-length RLE over both length lists at once, an optimal 7-bit code-length code.
        hlit / hdist / hclen are the header's counts (257.., 1.., 4..), written as given."""
        lf, df = token_freqs(tokens, eob)
        if llens is None:
            llens = limited_lengths(lf[:286], 15)
            n = 286
            while n > 257 and not llens[n - 1]:
                n -= 1
            llens = llens[:n]
        if dlens is None:
            f = df[:30]
            if sum(1 for x in f if x) < 2:
                f = list(f)
                f[0] = f[0] or 1
                if sum(1 for x in f if x) < 2:
                    f[1] = 1
            dlens = limited_lengths(f, 15)
            n = 30
            while n > 1 and not dlens[n - 1]:
                n -= 1
            dlens = dlens[:n]
        if rle is None:
            allowed = range(19) if cl_lens is None else [s for s in range(19) if cl_lens[s]]
            rle = rle_lengths(list(llens) + list(dlens), allowed)
        if cl_lens is None:
            cf = [0] * 19
            for s, _ in rle:
                cf[s] += 1
            if sum(1 for x in cf if x) < 2:
                cf[0 if not cf[0] else 1] = 1
            cl_lens = limited_lengths(cf, 7)
        if hclen is None:
            hclen = 19
            while hclen > 4 and not cl_lens[CLORDER[hclen - 1]]:
                hclen -= 1
        hlit = len(llens) if hlit is None else hlit
        hdist = len(dlens) if hdist is None else hdist
        w = self.w
        w.bits(1 if final else 0, 1)
        w.bits(2, 2)
        w.bits(hlit - 257, 5)
        w.bits(hdist - 1, 5)
        w.bits(hclen - 4, 4)
        for k in range(hclen):
            w.bits(cl_lens[CLORDER[k]], 3)
        cc = canonical(cl_lens)
        for s, x in rle:
            w.huff(cc[s] or 0, cl_lens[s])
            if s >= 16:
                w.bits(x, {16: 2, 17: 3, 18: 7}[s])
        full_l = list(llens) + [0] * (288 - len(llens))
        full_d = list(dlens) + [0] * (32 - len(dlens))
        lc, dc = canonical(full_l), canonical(full_d)
        write_tokens(w, tokens, [c or 0 for c in lc], full_l, [c or 0 for c in dc], full_d, eob)
        self.nout += sum(token_len(t) for t in tokens)

    def fill_to(self, bit, byte=0x41):
        """fixed blocks of literals up to bit position `bit` exactly (at least 73 bits away): 8-bit literals `byte`
        and 9-bit literals 0x90 set the phase"""
        d = bit - self.bit
        assert d >= 73, d
        while d > 73 + 8 * 4000:   # keep blocks short
            self.fixed([byte] * 4000)
            d = bit - self.bit
        d -= 10
        b = d % 8
        a = (d - 9 * b) // 8
        self.fixed([byte] * a + [0x90] * b)
        assert self.bit == bit


# ---------------------------------------------------------------------------------------------------- parsing
class _Table:
    """canonical decoding table: the low `bits` bits of the stream -> (symbol, length); None where no code is"""
    __slots__ = ("bits", "tab")

    def __init__(self, lengths):
        self.bits = max([l for l in lengths if l] or [1])
        tab = [None] * (1 << self.bits)
        for s, (l, c) in enumerate(zip(lengths, canonical(lengths))):
            if not l:
                continue
            r = int(format(c, "0%db" % l)[::-1], 2)
            e = (s, l)
            for k in range(r, 1 << self.bits, 1 << l):
                tab[k] = e
        self.tab = tab


_FIXED = None


class _Reader:
    __slots__ = ("data", "pos", "buf", "cnt")

    def __init__(self, data):
        self.data, self.pos, self.buf, self.cnt = data, 0, 0, 0

    def need(self, n):
        while self.cnt < n:
            if self.pos >= len(self.data):
                raise DeflateError("truncated")
            self.buf |= self.data[self.pos] << self.cnt
            self.pos += 1
            self.cnt += 8

    def bits(self, n):
        self.need(n)
        v = self.buf & ((1 << n) - 1)
        self.buf >>= n
        self.cnt -= n
        return v

    def bitpos(self):
        return self.pos * 8 - self.cnt

    def decode(self, t, what):
        # peek up to t.bits, zero-filled past the end; a code that reaches past the end is a truncation
        while self.cnt < t.bits and self.pos < len(self.data):
            self.buf |= self.data[self.pos] << self.cnt
            self.pos += 1
            self.cnt += 8
        e = t.tab[self.buf & ((1 << t.bits) - 1)]
        if e is None:
            raise DeflateError("invalid %s code" % what if self.cnt >= t.bits else "truncated")
        if e[1] > self.cnt:
            raise DeflateError("truncated")
        self.buf >>= e[1]
        self.cnt -= e[1]
        return e[0]


def parse(body, keep_tokens=True):
    """Decode a raw DEFLATE body.  Returns (output bytes, blocks, end bit).  Each block is a dict: type ('stored',
    'fixed', 'dynamic'), final, start / end bit, and for dynamic blocks hlit, hdist, hclen, llens, dlens, cllens
    (the code-length code, indexed by symbol) and rle ((sym, extra) pairs); for Huffman blocks `tokens`: ints for
    literals and (length, distance, length symbol) for matches.  Raises DeflateError where zlib's inflate fails."""
    global _FIXED
    r = _Reader(body)
    out = bytearray()
    blocks = []
    while True:
        start = r.bitpos()
        final = r.bits(1)
        btype = r.bits(2)
        blk = {"start": start, "final": final}
        if btype == 0:
            r.bits(r.cnt & 7)
            n, nn = r.bits(16), r.bits(16)
            if n != (~nn & 0xFFFF):
                raise DeflateError("invalid stored block lengths")
            assert r.cnt == 0
            if r.pos + n > len(body):
                raise DeflateError("truncated")
            out += body[r.pos:r.pos + n]
            r.pos += n
            blk.update(type="stored", len=n)
        elif btype == 3:
            raise DeflateError("invalid block type")
        else:
            if btype == 1:
                if _FIXED is None:
                    _FIXED = (_Table(FIXED_L), _Table(FIXED_D))
                lt, dt = _FIXED
                blk["type"] = "fixed"
            else:
                hlit, hdist, hclen = r.bits(5) + 257, r.bits(5) + 1, r.bits(4) + 4
                if hlit > 286 or hdist > 30:
                    raise DeflateError("too many length or distance symbols")
                cl = [0] * 19
                for k in range(hclen):
                    cl[CLORDER[k]] = r.bits(3)
                if not code_ok(cl, "codes"):
                    raise DeflateError("invalid code lengths set")
                ct = _Table(cl)
                lens, rle = [], []
                while len(lens) < hlit + hdist:
                    s = r.decode(ct, "code length")
                    if s < 16:
                        rle.append((s, 0))
                        lens.append(s)
                        continue
                    x = r.bits({16: 2, 17: 3, 18: 7}[s])
                    rle.append((s, x))
                    if s == 16:
                        if not lens:
                            raise DeflateError("invalid bit length repeat")
                        v, rep = lens[-1], 3 + x
                    else:
                        v, rep = 0, (3 + x if s == 17 else 11 + x)
                    if len(lens) + rep > hlit + hdist:
                        raise DeflateError("invalid bit length repeat")
                    lens += [v] * rep
                llens, dlens = lens[:hlit], lens[hlit:]
                if not llens[256]:
                    raise DeflateError("invalid code -- missing end-of-block")
                if not code_ok(llens, "lens"):
                    raise DeflateError("invalid literal/lengths set")
                if not code_ok(dlens, "dists"):
                    raise DeflateError("invalid distances set")
                lt = _Table(llens)
                dt = _Table(dlens) if any(dlens) else None
                blk.update(type="dynamic", hlit=hlit, hdist=hdist, hclen=hclen, llens=llens, dlens=dlens, cllens=cl,
                           rle=rle)
            toks = [] if keep_tokens else None
            while True:
                s = r.decode(lt, "literal/length")
                if s < 256:
                    out.append(s)
                    if keep_tokens:
                        toks.append(s)
                    continue
                if s == 256:
                    break
                if s > 285:
                    raise DeflateError("invalid literal/length code")
                length = LBASE[s - 257] + r.bits(LEXT[s - 257])
                if dt is None:
                    raise DeflateError("invalid distance code")
                ds = r.decode(dt, "distance")
                if ds > 29:
                    raise DeflateError("invalid distance code")
                dist = DBASE[ds] + r.bits(DEXT[ds])
                if dist > len(out):
                    raise DeflateError("invalid distance too far back")
                if dist >= length:
                    out += out[-dist:len(out) - dist + length]
                else:
                    pat = out[-dist:]
                    out += (pat * (length // dist + 1))[:length]
                if keep_tokens:
                    toks.append((length, dist, s))
            blk["tokens"] = toks
        blk["end"] = r.bitpos()
        blocks.append(blk)
        if final:
            return bytes(out), blocks, r.bitpos()


# ---------------------------------------------------------------------------------------------------- crafted corpus
# Streams with the features zlib never writes and the refusals next to them.  Each item is written at a nominal span
# start, a little before and a little after it, at every bit phase, behind filler that has no block-start candidates
# (fixed blocks), and behind 32 KB of stored output where it needs a full window.
def _bytes(n, seed):
    import random
    return random.Random(seed).randbytes(n)


def _window(s):
    """33 000 bytes of stored random output in 1 500-byte blocks"""
    data = _bytes(33000, 11)
    for i in range(0, len(data), 1500):
        s.stored(data[i:i + 1500])


def _all_syms(extra_lit=True):
    """every length symbol 257..285 and distance symbol 0..29, each at the bottom and top of its extra range, plus
    258 as 284 + 31"""
    lens = [v for i in range(29) for v in {LBASE[i], LBASE[i] + (1 << LEXT[i]) - 1}]
    dists = [v for i in range(30) for v in (DBASE[i], DBASE[i] + (1 << DEXT[i]) - 1)]
    toks = []
    for k in range(max(len(lens), len(dists))):
        toks.append((lens[k % len(lens)], dists[k % len(dists)]))
        if extra_lit:
            toks.append(0x30 + k % 40)
    return toks + [Raw(284, 31, *dist_sym(32768))]


def _far(s):
    return [(258, 32768)] + [(3 + k % 8, d) for k, d in enumerate(range(32507, 32769))] + \
        [Raw(284, 31, *dist_sym(32768)), Raw(284, 31, *dist_sym(32507))]


L9_EOB1 = [9] * 256 + [1]                                  # literals 9 bits, end-of-block 1 bit: complete
L9_SYMS = [9] * 256 + [6] * 28 + [5, 5]                    # literals, EOB and all 29 length symbols: complete
D_5x28_4x2 = [5] * 28 + [4, 4]                             # all 30 distance symbols: complete
L_CL7 = [8] * 148 + [9] * 108 + [7] * 24 + [8] * 6         # complete from the lengths 7, 8, 9 only
CL7 = [0] * 19
for _s, _l in {8: 1, 0: 2, 16: 3, 5: 4, 9: 5, 7: 6, 4: 7, 17: 7}.items():
    CL7[_s] = _l


def _deep_lens():
    """15-bit literal/length and distance codes: lengths 1..14, 15, 15"""
    ll = [0] * 258
    for k in range(14):
        ll[65 + k] = k + 1
    ll[256] = ll[257] = 15
    dl = [k + 1 for k in range(14)] + [15, 15]
    return ll, dl


def _deep_tokens():
    toks = []
    for k in range(14):
        toks += [65 + k] * (3 if k < 13 else 1)
        toks.append((3, DBASE[k]))
    return toks + [(3, DBASE[14]), (3, DBASE[15]), (3, DBASE[15] + 63)]


def _lit_text(n, seed):
    import random
    rng = random.Random(seed)
    return [rng.randrange(0x61, 0x7B) for _ in range(n)]


# name -> (needs the 32 KB window, item(stream) -> True when it ended the stream)
ITEMS = {
    # distances 32 507 .. 32 768, first thing in a span and through spans shorter than 32 KB
    "far_dynamic": (True, lambda s: s.dynamic(_far(s))),
    "far_fixed": (True, lambda s: s.fixed(_far(s))),
    # distance = bytes so far, and one more (zlib: too far back), in a later span
    "sofar": (False, lambda s: s.dynamic([(7, s.nout)] + _lit_text(20, 1))),
    "sofar_plus1": (False, lambda s: s.dynamic([(7, s.nout + 1)] + _lit_text(20, 1))),
    "sofar_plus1_fixed": (False, lambda s: s.fixed([(7, s.nout + 1)])),
    # every length and distance symbol
    "all_syms_fixed": (True, lambda s: s.fixed(_all_syms())),
    "all_syms_dynamic": (True, lambda s: s.dynamic(_all_syms())),   # HLIT 286, HDIST 30
    # code trees
    "one_dist_code": (False, lambda s: s.dynamic(_lit_text(30, 2) + [(5, 4), (9, 4), 0x41, (258, 4)],
                                                  dlens=[0, 0, 0, 1])),
    "one_dist_code_d1": (False, lambda s: s.dynamic(_lit_text(10, 3) + [(40, 1)], dlens=[1])),
    "empty_dist_tree": (False, lambda s: s.dynamic(_lit_text(50, 4), dlens=[0])),
    "eob_only": (False, lambda s: s.dynamic([], llens=[0] * 256 + [1], dlens=[0])),
    "hlit257_one_code": (False, lambda s: s.dynamic(_lit_text(40, 5), llens=L9_EOB1, dlens=[1])),
    "rep16_first_dist": (True, lambda s: s.dynamic(
        _lit_text(20, 6) + _all_syms(False), llens=L9_SYMS, dlens=D_5x28_4x2,
        rle=rle_lengths(L9_SYMS) + [(16, 3)] + rle_lengths(D_5x28_4x2[6:]))),
    "rep16_across": (True, lambda s: s.dynamic(_lit_text(20, 6) + _all_syms(False), llens=L9_SYMS,
                                               dlens=D_5x28_4x2)),
    "rep18_across": (False, lambda s: s.dynamic(
        _lit_text(20, 7) + [(3, 40), (3, 60), (3, 33)], llens=[9] * 256 + [2, 2] + [0] * 28,
        dlens=[0] * 10 + [1, 1])),
    "rep17_across": (False, lambda s: s.dynamic(
        _lit_text(20, 8) + [(3, 5), (3, 7)], llens=[9] * 256 + [2, 2, 0, 0], dlens=[0, 0, 0, 1, 1])),
    "hclen5": (False, lambda s: s.dynamic(_lit_text(60, 9), llens=[8] * 255 + [0, 8], dlens=[0],
                                          cl_lens=[3, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 2, 4, 4])),
    "hclen19": (False, lambda s: s.dynamic(_lit_text(60, 10) + [(10, 3)], hclen=19)),
    "deep15": (False, lambda s: s.dynamic(_deep_tokens(), llens=_deep_lens()[0], dlens=_deep_lens()[1])),
    "cl7": (True, lambda s: s.dynamic(_all_syms(), llens=L_CL7, dlens=D_5x28_4x2, cl_lens=CL7)),
    # block mix
    "stored_len0": (False, lambda s: s.stored(b"")),
    "stored_len65535": (False, lambda s: s.stored(_bytes(65535, 12))),
    "stored_final_padded": (False, lambda s: s.stored(_bytes(3000, 13), final=True) or True),
    "stored_nonzero_padding": (False, lambda s: s.stored(_bytes(3000, 14), pad=0xFF)),
    # refusals
    "fixed_286": (False, lambda s: s.fixed(_lit_text(5, 15) + [Raw(286)])),
    "fixed_287": (False, lambda s: s.fixed(_lit_text(5, 15) + [Raw(287)])),
    "fixed_dist30": (False, lambda s: s.fixed(_lit_text(5, 16) + [Raw(257, 0, 30)])),
    "fixed_dist31": (False, lambda s: s.fixed(_lit_text(5, 16) + [Raw(257, 0, 31)])),
    "over_lit": (False, lambda s: s.dynamic(_lit_text(40, 17), llens=[8] + L9_EOB1[1:], dlens=[1])),
    "incomplete_lit": (False, lambda s: s.dynamic(_lit_text(40, 17), llens=L9_EOB1[:255] + [0, 1], dlens=[1])),
    "over_dist": (False, lambda s: s.dynamic(_lit_text(10, 18) + [(3, 1)], dlens=[1, 1, 1])),
    "incomplete_dist": (False, lambda s: s.dynamic(_lit_text(10, 18) + [(3, 1)], dlens=[1, 2])),
    "over_cl": (False, lambda s: s.dynamic(_lit_text(60, 9), llens=[8] * 255 + [0, 8], dlens=[0],
                                           cl_lens=[3, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 2, 3, 4])),
    "incomplete_cl": (False, lambda s: s.dynamic(_lit_text(60, 9), llens=[8] * 255 + [0, 8], dlens=[0],
                                                 cl_lens=[3, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 2, 4, 5])),
    "one_cl_code": (False, lambda s: s.dynamic([], llens=[0] * 256 + [1], dlens=[0],
                                               cl_lens=[0] * 18 + [1], rle=[(18, 127), (18, 127)])),
    "missing_eob_len": (False, lambda s: s.dynamic(_lit_text(40, 19), llens=[8] * 256 + [0], dlens=[0], eob=False)),
    "hclen4": (False, lambda s: s.dynamic([], llens=[0] * 257, dlens=[0], cl_lens=[1] + [0] * 17 + [1], hclen=4,
                                          eob=False)),
    "hlit287": (False, lambda s: s.dynamic(_lit_text(10, 20), llens=L9_EOB1 + [0] * 30, dlens=[1])),
    "hdist31": (False, lambda s: s.dynamic(_lit_text(10, 20), llens=L9_EOB1, dlens=[1] + [0] * 30)),
    "rep16_at_start": (False, lambda s: s.dynamic(_lit_text(10, 21), llens=L9_EOB1, dlens=[1],
                                                  rle=[(16, 0)] + rle_lengths(L9_EOB1 + [1])[1:])),
    "rep_overrun": (False, lambda s: s.dynamic(_lit_text(10, 22), llens=[9] * 256 + [2, 2] + [0] * 28,
                                               dlens=[0] * 10 + [1, 1],
                                               rle=rle_lengths([9] * 256 + [2, 2]) + [(18, 38 - 11 + 1), (1, 0),
                                                                                       (1, 0)])),
    "btype3": (False, lambda s: s.w.bits(7, 3)),
    "missing_eob_end": (False, lambda s: s.fixed(_lit_text(40, 23), final=True, eob=False) or True),
}


def place(name, delta, phase, span=8192):
    """item `name` at byte `delta` from a nominal span start (a multiple of `span` bytes), at bit phase `phase`"""
    window, item = ITEMS[name]
    s = Stream()
    if window:
        _window(s)
    base = -(-(s.bit + 200) // (span * 8)) * span * 8
    s.fill_to(base + delta * 8 + phase)
    if not item(s):
        s.fixed(_lit_text(30, 24) + [(12, 9)], final=True)
    return s.body()


def crafted(deltas=(-3, 0, 5), phases=range(8), names=None):
    """(name, body) over the items placed at every delta and phase, plus the unplaced streams"""
    out = []
    for name in names or ITEMS:
        for d in deltas:
            for p in phases:
                out.append(("%s@%+d.%d" % (name, d, p), place(name, d, p)))
    return out + unplaced()


def unplaced():
    out = []
    # distance = bytes so far (valid) and one more, in span 0
    for extra, tag in ((0, "sofar_span0"), (1, "sofar_plus1_span0")):
        s = Stream()
        s.fixed(_lit_text(100, 25))
        s.dynamic([(6, s.nout + extra)] + _lit_text(5, 25), final=True)
        out.append((tag, s.body()))
    # a long run of fixed blocks only, with matches: no span after the first has a candidate
    s = Stream()
    for k in range(3000):
        s.fixed(_lit_text(6, k) + [(3 + k % 50, 1 + k % 6)], final=k == 2999)
    out.append(("fixed_only_run", s.body()))
    # the biggest stored block, final
    s = Stream()
    s.stored(_bytes(65535, 26), final=True)
    out.append(("stored_65535_final", s.body()))
    out.append(("far_chain", far_chain()))
    return out


def far_chain(n=8):
    """n x (32 KB stored block, then a fixed block of distance-32 768 matches)"""
    s = Stream()
    for k in range(n):
        s.stored(_bytes(32768, 100 + k))
        s.fixed([(258, 32768), (100, 32768), (3, 32768)] + _lit_text(10, k), final=k == n - 1)
    return s.body()
