// inflate_core.cuh -- the raw-DEFLATE (RFC 1951) decoding core shared by the inflate kernels (inflate.cu), the host
// chain logic of lb2_inflate_run (api.cu) and the CPU emulator of the tests (tests/emu/inflate_emu.cpp).
//
// Speculative parallel inflate (the approach of pugz and rapidgzip): the compressed body is cut into nominal spans of
// S bytes.  Span 0 starts at bit 0; every other span starts at the first block-header candidate at or after its
// nominal start (find_candidate).  One decoder per span counts the span's output (decode_span<false>) and stops at the
// first dynamic or stored block whose key is at or after the next span's nominal start.  Chain accepts a span only if
// its start key is the end key of the span before it; a rejected span is counted again from that known-true key.  The
// confirmed spans are then decoded (decode_span<true>) into a u16 arena where 0x8000 | w stands for byte w of the
// unknown 32 KB window before the span, which the resolve kernels fill in from the spans before.
//
// Keys.  A candidate's key orders block starts: bit << 2 for a block whose header is read at `bit` (dynamic blocks,
// and span 0's first block of any type); (bit << 2) | 2 | BFINAL for a stored block whose LEN field starts at `bit`
// (the header bits and padding in front of it may sit at several offsets, which all decode the same).
//
// Seek table.  A stream whose writer recorded where its blocks start (the GPU writers end every 64 KB chunk
// byte-aligned with an empty stored block and can keep each run of chunks' compressed and decoded lengths, see
// seek_table.py) needs no search: Table turns the entries into one exact-stop span each, decoded once straight into
// the arena, and accepts the results only if they chain as Chain::walk requires.  A refused table costs one decode
// pass; the caller then runs the search above on the same stream.
#pragma once
#include <cstdint>
#include <utility>
#include <vector>

#ifdef __CUDACC__
#define IFL_HD __host__ __device__ __forceinline__
#else
#define IFL_HD inline
#endif

namespace lb2 {
namespace ifl {

constexpr uint64_t KEY_NONE = ~0ull;
constexpr uint32_t GIVE_UP_SPANS = 4;  // an unconfirmed span gives up this many span sizes past its end
IFL_HD uint64_t key_header(uint64_t bit) { return bit << 2; }
IFL_HD uint64_t key_stored(uint64_t len_bit, uint32_t bfinal) { return (len_bit << 2) | 2u | bfinal; }
IFL_HD uint64_t key_bit(uint64_t key) { return key >> 2; }
IFL_HD bool key_is_stored(uint64_t key) { return (key & 2) != 0; }

// span status
enum : int32_t {
  ST_OK = 0,
  ST_BAD_HEADER = -1,   // BTYPE 3, or a dynamic header zlib refuses
  ST_BAD_CODE = -2,     // a code that is not in the table (or length / distance symbol out of range)
  ST_BAD_DIST = -3,     // distance further back than the data before it
  ST_BAD_STORED = -4,   // LEN != ~NLEN
  ST_EOF = -5,          // ran past the end of the input
  ST_GIVE_UP = -6,      // an unconfirmed span ran the give-up distance past its end
  ST_OVERFLOW = -7,     // decode pass: more output than the count pass measured
  ST_PAST_STOP = -8     // exact stop: a block header beyond stop_bit
};

// ---- tables -------------------------------------------------------------------------------------------------------
static const uint16_t h_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99,
                                     115, 131, 163, 195, 227, 258};
static const uint8_t h_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t h_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025,
                                     1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint8_t h_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
static const uint8_t h_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
#ifdef __CUDACC__
static __constant__ uint16_t d_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83,
                                            99, 115, 131, 163, 195, 227, 258};
static __constant__ uint8_t d_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static __constant__ uint16_t d_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769,
                                            1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static __constant__ uint8_t d_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
static __constant__ uint8_t d_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
#endif
#ifdef __CUDA_ARCH__
#define IFL_T(name) d_##name
#else
#define IFL_T(name) h_##name
#endif

IFL_HD uint8_t load_byte(const uint8_t *p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// ---- bit reader: LSB first; every load is bounded by n, bytes past it read as zero and pos() tells how far it went --
struct Bits {
  const uint8_t *p;
  uint64_t n;      // input bytes
  uint64_t next;   // next byte to load
  uint64_t buf;
  uint32_t cnt;    // valid bits in buf
  IFL_HD void refill() {
    while (cnt <= 56) {
      const uint64_t b = next < n ? load_byte(p + next) : 0;
      buf |= b << cnt;
      next++;
      cnt += 8;
    }
  }
  IFL_HD void init(const uint8_t *in, uint64_t n_bytes, uint64_t bit) {
    p = in; n = n_bytes; next = bit >> 3; buf = 0; cnt = 0;
    refill();
    drop((uint32_t)(bit & 7));
  }
  IFL_HD uint64_t pos() const { return next * 8 - cnt; }
  IFL_HD bool over() const { return pos() > n * 8; }
  IFL_HD uint32_t peek(uint32_t k) const { return (uint32_t)(buf & ((1ull << k) - 1)); }
  IFL_HD void drop(uint32_t k) { buf >>= k; cnt -= k; }
  IFL_HD uint32_t get(uint32_t k) {  // k <= 32
    if (cnt < k) refill();
    const uint32_t v = peek(k);
    drop(k);
    return v;
  }
};

// ---- canonical Huffman decoding: counts + symbols (RFC 1951 3.2.2) and a LUT for codes of up to B bits ------------------
template <int N, int B> struct Huff {
  uint16_t count[16];   // codes per length (count[0] = 0)
  uint16_t sym[N];      // symbols ordered by code
  uint16_t lut[1 << B]; // low B bits of the stream -> (length << 9) | symbol, 0 = longer code or none
};
constexpr int LUT_LIT = 9, LUT_DIST = 8;
typedef Huff<288, LUT_LIT> HuffL;
typedef Huff<32, LUT_DIST> HuffD;

// What zlib's inflate_table accepts (kind 0: code-length code, 1: literal/length, 2: distance): never
// over-subscribed; incomplete only for a literal/length or distance code whose one code has length 1; no codes at all
// only for distances.  (zlib builds an all-invalid code-length table when it has no codes; every length then decodes
// as 0, symbol 256 gets no code and the header is refused, so refusing it here is the same outcome.)
IFL_HD bool code_ok(const uint16_t *count, int kind) {
  int max = 15;
  while (max >= 1 && count[max] == 0) max--;
  if (max == 0) return kind == 2;
  int left = 1;
  for (int len = 1; len <= 15; len++) {
    left <<= 1;
    left -= count[len];
    if (left < 0) return false;
  }
  return !(left > 0 && (kind == 0 || max != 1));
}

template <int N, int B> IFL_HD void huff_build(Huff<N, B> &h, const uint8_t *len, int n) {
  for (int i = 0; i < 16; i++) h.count[i] = 0;
  for (int s = 0; s < n; s++) h.count[len[s]]++;
  h.count[0] = 0;
  uint16_t offs[16];
  offs[1] = 0;
  for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + h.count[l];
  for (int s = 0; s < n; s++)
    if (len[s]) h.sym[offs[len[s]]++] = (uint16_t)s;
  for (int i = 0; i < (1 << B); i++) h.lut[i] = 0;
  uint32_t code = 0, idx = 0;
  for (int l = 1; l <= B; l++) {
    for (uint32_t k = 0; k < h.count[l]; k++, code++) {
      uint32_t rev = 0;
      for (int j = 0; j < l; j++) rev |= ((code >> j) & 1) << (l - 1 - j);
      const uint16_t e = (uint16_t)((l << 9) | h.sym[idx++]);
      for (uint32_t r = rev; r < (1u << B); r += 1u << l) h.lut[r] = e;
    }
    code <<= 1;
  }
}

// next symbol, or -1 for a code the table does not have; b must hold >= 15 bits
template <int N, int B> IFL_HD int huff_decode(const Huff<N, B> &h, Bits &b) {
  const uint32_t e = h.lut[b.peek(B)];
  if (e) {
    b.drop(e >> 9);
    return (int)(e & 511);
  }
  const uint32_t bits = b.peek(15);
  int code = 0, first = 0, index = 0;
  for (int len = 1; len <= 15; len++) {
    code |= (bits >> (len - 1)) & 1;
    const int count = h.count[len];
    if (code - first < count) {
      b.drop(len);
      return h.sym[index + code - first];
    }
    index += count;
    first += count;
    first <<= 1;
    code <<= 1;
  }
  return -1;
}

// ---- dynamic block header ---------------------------------------------------------------------------------------
struct HdrScratch {
  uint16_t lcount[16], dcount[16];
  uint8_t cllen[20];
  HuffD cl;
};

// Reads HLIT, HDIST, HCLEN, the code-length code and the code lengths (b just past BTYPE) and checks them by zlib's
// rules.  lens (may be null) receives the nlen literal/length then the ndist distance lengths.  The block decoder and
// the candidate filter both run this, so the filter refuses no header the decoder accepts.
IFL_HD int32_t read_dynamic(Bits &b, HdrScratch &s, uint8_t *lens, uint32_t &nlen, uint32_t &ndist) {
  b.refill();
  nlen = b.get(5) + 257;
  ndist = b.get(5) + 1;
  const uint32_t ncode = b.get(4) + 4;
  if (nlen > 286 || ndist > 30) return ST_BAD_HEADER;
  for (int i = 0; i < 19; i++) s.cllen[i] = 0;
  for (uint32_t k = 0; k < ncode; k++) s.cllen[IFL_T(clorder)[k]] = (uint8_t)b.get(3);
  huff_build(s.cl, s.cllen, 19);
  if (!code_ok(s.cl.count, 0)) return ST_BAD_HEADER;
  for (int i = 0; i < 16; i++) s.lcount[i] = s.dcount[i] = 0;
  const uint32_t total = nlen + ndist;
  uint32_t i = 0, prev = 0;
  bool eob = false;
  while (i < total) {
    if (b.cnt < 24) b.refill();
    const int sym = huff_decode(s.cl, b);
    if (sym < 0) return ST_BAD_HEADER;
    uint32_t len, rep;
    if (sym < 16) { len = (uint32_t)sym; rep = 1; }
    else if (sym == 16) { if (i == 0) return ST_BAD_HEADER; len = prev; rep = 3 + b.get(2); }
    else if (sym == 17) { len = 0; rep = 3 + b.get(3); }
    else { len = 0; rep = 11 + b.get(7); }
    if (i + rep > total) return ST_BAD_HEADER;
    if (i <= 256 && 256 < i + rep && len) eob = true;
    const uint32_t in_lit = i < nlen ? (nlen - i < rep ? nlen - i : rep) : 0;
    s.lcount[len] += (uint16_t)in_lit;
    s.dcount[len] += (uint16_t)(rep - in_lit);
    if (lens)
      for (uint32_t k = 0; k < rep; k++) lens[i + k] = (uint8_t)len;
    i += rep;
    prev = len;
  }
  if (b.over()) return ST_EOF;
  if (!eob) return ST_BAD_HEADER;
  s.lcount[0] = s.dcount[0] = 0;
  if (!code_ok(s.lcount, 1) || !code_ok(s.dcount, 2)) return ST_BAD_HEADER;
  return ST_OK;
}

// ---- candidate filter -------------------------------------------------------------------------------------------
// a dynamic-block header zlib would accept starts at bit p
IFL_HD bool dynamic_candidate(const uint8_t *in, uint64_t n, uint64_t p, HdrScratch &s) {
  if (p + 17 > n * 8) return false;
  Bits b;
  b.init(in, n, p);
  if ((b.peek(3) >> 1) != 2) return false;
  const uint32_t hl = (b.buf >> 3) & 31, hd = (b.buf >> 8) & 31;
  if (hl > 29 || hd > 29) return false;
  b.drop(3);
  uint32_t nl, nd;
  return read_dynamic(b, s, nullptr, nl, nd) == ST_OK;
}

// LEN == ~NLEN at byte `at`, and the block's bytes end inside the input
IFL_HD bool stored_len_ok(const uint8_t *in, uint64_t n, uint64_t at) {
  if (at + 4 > n) return false;
  const uint32_t len = load_byte(in + at) | (uint32_t)load_byte(in + at + 1) << 8;
  const uint32_t nlen = load_byte(in + at + 2) | (uint32_t)load_byte(in + at + 3) << 8;
  return len == (~nlen & 0xFFFFu) && at + 4 + len <= n;
}

// the 3 header bits at bit q start a block zlib could read: not BTYPE 3; a dynamic header it accepts; a stored
// block whose LEN / NLEN agree
IFL_HD bool next_header_ok(const uint8_t *in, uint64_t n, uint64_t q, HdrScratch &s) {
  if (q + 3 > n * 8) return false;
  Bits b;
  b.init(in, n, q);
  const uint32_t t = b.peek(3) >> 1;
  if (t == 3) return false;
  if (t == 1) return true;
  if (t == 2) return dynamic_candidate(in, n, q, s);
  return stored_len_ok(in, n, (q + 3 + 7) >> 3);
}

// Key of a stored block whose LEN field is at byte-aligned bit p, or KEY_NONE.  The header and padding in front of
// LEN must be zero bits (zlib writes them so): z zero bits right below p, z >= 2.  z == 2 leaves one reading, the
// header at p - 3 with BFINAL 1.  Otherwise the block is taken as not final, and the block after it must have a
// header zlib could read, which rejects most chance LEN / NLEN matches in compressed data.
IFL_HD uint64_t stored_candidate(const uint8_t *in, uint64_t n, uint64_t p, HdrScratch &s) {
  const uint64_t at = p >> 3;
  if ((p & 7) || at < 2 || !stored_len_ok(in, n, at)) return KEY_NONE;
  const uint32_t below = (uint32_t)load_byte(in + at - 1) << 8 | load_byte(in + at - 2);  // bits p-16 .. p-1
  uint32_t z = 0;
  while (z < 10 && !((below >> (15 - z)) & 1)) z++;
  if (z < 2) return KEY_NONE;
  if (z == 2) return key_stored(p, 1);
  const uint32_t len = load_byte(in + at) | (uint32_t)load_byte(in + at + 1) << 8;
  return next_header_ok(in, n, p + 32 + 8ull * len, s) ? key_stored(p, 0) : KEY_NONE;
}

// the first candidate key at or after bit `from` and before bit `to`
IFL_HD uint64_t candidate_at(const uint8_t *in, uint64_t n, uint64_t p, HdrScratch &s) {
  if (dynamic_candidate(in, n, p, s)) return key_header(p);
  if ((p & 7) == 0) return stored_candidate(in, n, p, s);
  return KEY_NONE;
}
IFL_HD uint64_t find_candidate(const uint8_t *in, uint64_t n, uint64_t from, uint64_t to, HdrScratch &s) {
  for (uint64_t p = from; p < to; p++) {
    const uint64_t k = candidate_at(in, n, p, s);
    if (k != KEY_NONE) return k;
  }
  return KEY_NONE;
}

// ---- span decoder -----------------------------------------------------------------------------------------------
struct SpanJob {
  uint64_t start_key;
  uint64_t stop_bit;   // stop at the first dynamic / stored block (after the first) whose key is at or after this bit
  uint64_t limit_bit;  // give up once the input position passes this bit (KEY_NONE: confirmed start, no cap)
  uint64_t out_off;    // decode pass: where the span's output starts in the arena
  uint64_t out_len;    // decode pass: the counted length
  uint32_t first;      // span 0: no window in front of it
  uint32_t exact;      // stop at the block header (of any type) read exactly at stop_bit; one beyond it is an error
  // where the span's stream is: the kernels decode in[in_off .. in_off + in_n); out_base is the stream's first output
  // byte in the arena (a window marker must not point before it); member indexes the per-stream status
  uint64_t in_off, in_n, out_base;
  uint32_t member, pad2;
};
struct SpanResult {
  uint64_t end_key;    // key where the span stopped (KEY_NONE after the final block)
  uint64_t out_len;
  uint64_t end_bit;    // input bit position where the span stopped
  int32_t status;
  uint32_t final;      // the final block was decoded
};
struct DecodeState {
  HuffL lit;
  HuffD dist;
  HdrScratch hs;
  uint8_t lens[320];
};

IFL_HD void fixed_tables(DecodeState &st) {
  for (int i = 0; i < 288; i++) st.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
  huff_build(st.lit, st.lens, 288);
  for (int i = 0; i < 30; i++) st.lens[i] = 5;
  huff_build(st.dist, st.lens, 30);
}

// Decodes one span from job.start_key.  EMIT = false counts the output; EMIT = true writes it to out[0 .. job.out_len)
// as u16: bytes, or 0x8000 | w for byte w of the 32 KB before the span.  T = uint8_t is the byte-output variant for a
// stream decoded whole by one decoder (job.first = 1: no window, so no markers); more or fewer bytes than job.out_len
// give ST_OVERFLOW.
template <class T> struct NoDeduce { typedef T type; };  // the output type is named, never deduced (out may be nullptr)
template <bool EMIT, class T = uint16_t>
IFL_HD void decode_span(const uint8_t *in, uint64_t n, const SpanJob &job, DecodeState &st, typename NoDeduce<T>::type *out,
                        SpanResult &res) {
  Bits b;
  const uint64_t start = key_bit(job.start_key);
  b.init(in, n, start);
  const uint64_t cap = EMIT ? job.out_len : ~0ull;
  const uint64_t window = job.first ? 0 : 32768;
  uint64_t pos = 0;
  int32_t status = ST_OK;
  uint64_t end_key = KEY_NONE;
  uint32_t final = 0, tables = 0;  // tables: 0 none, 1 fixed, 2 dynamic
  bool first_block = true;
  for (;;) {
    uint32_t bfinal, btype;
    if (first_block && key_is_stored(job.start_key)) {
      bfinal = (uint32_t)(job.start_key & 1);
      btype = 0;
    } else {
      const uint64_t hb = b.pos();
      if (hb + 3 > n * 8) { status = ST_EOF; break; }
      const uint32_t h = b.peek(3);
      if (!first_block && job.exact) {
        if (hb == job.stop_bit) { end_key = key_header(hb); break; }
        if (hb > job.stop_bit) { status = ST_PAST_STOP; break; }
      } else if (!first_block) {
        if ((h >> 1) == 2 && hb >= job.stop_bit) { end_key = key_header(hb); break; }
        if ((h >> 1) == 0) {
          const uint64_t lb = (hb + 3 + 7) & ~7ull;
          if (lb >= job.stop_bit) { end_key = key_stored(lb, h & 1); break; }
        }
      }
      b.drop(3);
      bfinal = h & 1;
      btype = h >> 1;
      if (btype == 0) b.drop((uint32_t)((8 - (b.pos() & 7)) & 7));
    }
    first_block = false;
    if (btype == 0) {
      const uint32_t len = b.get(16), nlen = b.get(16);
      if (len != (~nlen & 0xFFFFu)) { status = ST_BAD_STORED; break; }
      const uint64_t at = b.pos() >> 3;  // byte aligned here
      if (at + len > n) { status = ST_EOF; break; }
      if (EMIT) {
        if (pos + len > cap) { status = ST_OVERFLOW; break; }
        for (uint32_t k = 0; k < len; k++) out[pos + k] = load_byte(in + at + k);
      }
      b.init(in, n, (at + len) * 8);
      pos += len;
    } else if (btype == 3) {
      status = ST_BAD_HEADER;
      break;
    } else {
      if (btype == 1) {
        if (tables != 1) { fixed_tables(st); tables = 1; }
      } else {
        uint32_t nl, nd;
        status = read_dynamic(b, st.hs, st.lens, nl, nd);
        if (status != ST_OK) break;
        huff_build(st.lit, st.lens, (int)nl);
        huff_build(st.dist, st.lens + nl, (int)nd);
        tables = 2;
      }
      for (;;) {
        if (b.cnt < 48) b.refill();
        const int sym = huff_decode(st.lit, b);
        if (sym < 0) { status = ST_BAD_CODE; break; }
        if (sym < 256) {
          if (EMIT) {
            if (pos >= cap) { status = ST_OVERFLOW; break; }
            out[pos] = (uint16_t)sym;
          }
          pos++;
        } else if (sym == 256) {
          break;
        } else {
          const int ls = sym - 257;
          if (ls >= 29) { status = ST_BAD_CODE; break; }
          const uint32_t len = IFL_T(lbase)[ls] + b.get(IFL_T(lext)[ls]);
          const int ds = huff_decode(st.dist, b);
          if (ds < 0 || ds >= 30) { status = ST_BAD_CODE; break; }
          const uint32_t dist = IFL_T(dbase)[ds] + b.get(IFL_T(dext)[ds]);
          if (dist > pos + window) { status = ST_BAD_DIST; break; }
          if (EMIT) {
            if (pos + len > cap) { status = ST_OVERFLOW; break; }
            const int64_t src = (int64_t)pos - (int64_t)dist;
            uint32_t j = 0;
            for (uint32_t k = 0; k < len; k++) {  // repeats the last `dist` values when the match overlaps itself
              const int64_t s = src + j;
              out[pos + k] = s < 0 ? (T)(0x8000u | (uint32_t)(32768 + s)) : out[s];
              if (++j == dist) j = 0;
            }
          }
          pos += len;
        }
        if (b.over()) { status = ST_EOF; break; }
        if (b.pos() > job.limit_bit) { status = ST_GIVE_UP; break; }
      }
      if (status != ST_OK) break;
    }
    if (b.over()) { status = ST_EOF; break; }
    if (b.pos() > job.limit_bit) { status = ST_GIVE_UP; break; }
    if (bfinal) { final = 1; break; }
  }
  if (EMIT && status == ST_OK && pos != cap) status = ST_OVERFLOW;
  res.end_key = end_key;
  res.out_len = pos;
  res.end_bit = b.pos();
  res.status = status;
  res.final = final;
}

// ---- resolve: the value of output position i of a span whose output starts at `off` in the final arena -----------
// Returns false for a window position before the stream start `base` (corrupt data).
IFL_HD bool resolve_value(uint16_t v, uint64_t off, const uint8_t *final_out, uint8_t &byte, uint64_t base = 0) {
  if (!(v & 0x8000)) { byte = (uint8_t)v; return true; }
  const uint64_t w = v & 0x7FFF;
  if (off + w < base + 32768) { byte = 0; return false; }
  byte = final_out[off + w - 32768];
  return true;
}

// ---- chain (host) -----------------------------------------------------------------------------------------------
// Spans are used only if their start key is the end key of the span before them, back to bit 0.  Rounds: count the
// spans that need it, walk the chain as far as the results agree, and give the first disagreeing span the known-true
// start (counted again in the next round, without the give-up cap).  Every round confirms at least one more span.
struct Chain {
  uint64_t n_bytes = 0;
  std::vector<SpanJob> job;     // one per active span (span 0 and every nominal span with a candidate)
  std::vector<SpanResult> res;
  std::vector<uint8_t> counted;
  std::vector<uint8_t> moved;   // the span's candidate has been replaced
  size_t next = 0;              // first span not yet accepted
  uint64_t prev_end = 0;        // end key of the last accepted span
  uint32_t n_nominal = 0, n_absorbed = 0, n_rejected = 0, n_rounds = 0;
  bool done = false;
  int32_t error = ST_OK;

  // cand[k]: the candidate key of nominal span k >= 1 (cand[0] is ignored); giveup: multiple of the span size;
  // the stream is in[in_off .. in_off + n) of the kernels' input, `member` its index in a member table
  void init(const uint64_t *cand, uint32_t n_spans, uint64_t span_bytes, uint64_t n, uint32_t giveup, uint64_t in_off = 0,
            uint32_t member = 0) {
    n_bytes = n;
    n_nominal = n_spans;
    std::vector<uint64_t> nominal{0};
    std::vector<uint64_t> start{key_header(0)};
    for (uint32_t k = 1; k < n_spans; k++) {
      if (cand[k] == KEY_NONE) { n_absorbed++; continue; }
      nominal.push_back((uint64_t)k * span_bytes * 8);
      start.push_back(cand[k]);
    }
    job.resize(start.size());
    for (size_t i = 0; i < start.size(); i++) {
      SpanJob &j = job[i];
      j.start_key = start[i];
      j.stop_bit = i + 1 < start.size() ? nominal[i + 1] : KEY_NONE;
      const uint64_t end = i + 1 < start.size() ? nominal[i + 1] : n * 8;
      j.limit_bit = i == 0 ? KEY_NONE : end + (uint64_t)giveup * span_bytes * 8;
      j.out_off = j.out_len = 0;
      j.first = i == 0;
      j.exact = 0;
      j.in_off = in_off;
      j.in_n = n;
      j.out_base = 0;
      j.member = member;
      j.pad2 = 0;
    }
    res.assign(job.size(), SpanResult{});
    counted.assign(job.size(), 0);
    moved.assign(job.size(), 0);
  }
  // spans to count in the next round
  std::vector<uint32_t> pending() const {
    std::vector<uint32_t> p;
    if (done || error) return p;
    for (size_t i = next; i < job.size(); i++)
      if (!counted[i]) p.push_back((uint32_t)i);
    return p;
  }
  void set_result(uint32_t i, const SpanResult &r) { res[i] = r; counted[i] = 1; }
  void reject(size_t i, uint64_t start) {
    if (!moved[i]) n_rejected++;
    moved[i] = 1;
    job[i].start_key = start;
    counted[i] = 0;
  }
  void advance() {
    n_rounds++;
    walk();
    // Further on, a span whose start differs from where the span before it ended (by that span's own, still
    // unconfirmed, result) is counted again from there in the same round, under the give-up cap.  The walk above
    // still accepts it only once the span before it is confirmed with that end, so the rejections of one round are
    // resolved together instead of one per round.
    if (done || error) return;
    for (size_t j = next + 1; j < job.size(); j++)
      if (counted[j] && counted[j - 1] && res[j - 1].status == ST_OK && !res[j - 1].final &&
          job[j].start_key != res[j - 1].end_key)
        reject(j, res[j - 1].end_key);
  }
  void walk() {
    while (!done && !error && next < job.size()) {
      if (!counted[next]) return;
      const SpanResult &r = res[next];
      if (next > 0 && job[next].start_key != prev_end) {  // a false candidate, or the true block lies beyond it
        reject(next, prev_end);
        job[next].limit_bit = KEY_NONE;
        return;
      }
      if (r.status != ST_OK) {
        if (job[next].limit_bit == KEY_NONE) { error = r.status; return; }
        job[next].limit_bit = KEY_NONE;  // a true start that gave up: count it again without the cap
        counted[next] = 0;
        return;
      }
      prev_end = r.end_key;
      if (r.final) {
        done = true;
        job.resize(next + 1);
        res.resize(next + 1);
        return;
      }
      next++;
    }
    if (!done && !error && next == job.size()) error = ST_EOF;
  }
  // after done: output offsets of the confirmed spans, from `base` in the arena; returns the stream's total output
  uint64_t layout(uint64_t base = 0) {
    uint64_t off = 0;
    for (size_t i = 0; i < job.size(); i++) {
      job[i].out_off = base + off;
      job[i].out_len = res[i].out_len;
      job[i].limit_bit = KEY_NONE;
      job[i].out_base = base;
      off += res[i].out_len;
    }
    return off;
  }
  uint64_t in_bytes() const { return job.empty() ? 0 : (res.back().end_bit + 7) / 8; }
};

// ---- seek table (host) -------------------------------------------------------------------------------------------
// Entry e covers in[in_len of the entries before it .. + e.in_len) and decodes to e.out_len bytes; every entry after
// the first starts with a block header at its first byte.  The entries come from outside the program, so init refuses
// any that could not describe the stream: a zero length, more than MAX_RATIO output bytes per input byte (258-byte
// matches of 2 bits each), or more input than the n bytes there are.  A refused init allocates nothing.
constexpr uint64_t MAX_RATIO = 1032;
struct TableEntry {
  uint64_t in_len, out_len;
};
struct Table {
  std::vector<SpanJob> job;
  uint64_t in_total = 0, out_total = 0;

  // the stream is in[in_off .. in_off + n) of the kernels' input, its output starts at out_base of the arena
  bool init(const TableEntry *e, uint32_t n_entries, uint64_t n, uint64_t in_off = 0, uint64_t out_base = 0,
            uint32_t member = 0) {
    job.clear();
    in_total = out_total = 0;
    if (!n_entries) return false;
    for (uint32_t i = 0; i < n_entries; i++) {
      if (!e[i].in_len || !e[i].out_len || e[i].in_len > n - in_total || (e[i].out_len - 1) / MAX_RATIO >= e[i].in_len ||
          e[i].out_len > ~0ull / 4 - out_total)
        return false;
      in_total += e[i].in_len;
      out_total += e[i].out_len;
    }
    job.resize(n_entries);
    uint64_t in = 0, out = 0;
    for (uint32_t i = 0; i < n_entries; i++) {
      const uint64_t end = (in + e[i].in_len) * 8;
      job[i] = SpanJob{key_header(in * 8), i + 1 < n_entries ? end : KEY_NONE, end, out_base + out, e[i].out_len,
                       i == 0, 1, in_off, n, out_base, member, 0};
      in += e[i].in_len;
      out += e[i].out_len;
    }
    return true;
  }
  // The chain argument of Chain::walk: every span decoded exactly its length and stopped at the header the next one
  // starts from, only the last one decoded the final block and it ended with the table's last byte.  Accepted spans
  // are therefore the serial decode of the stream cut at the table's boundaries.
  bool accept(const SpanResult *r) const {
    for (size_t i = 0; i < job.size(); i++) {
      const bool last = i + 1 == job.size();
      if (r[i].status != ST_OK || r[i].out_len != job[i].out_len || r[i].final != (last ? 1u : 0u)) return false;
      if (!last && r[i].end_key != job[i + 1].start_key) return false;
      if (last && (r[i].end_bit + 7) / 8 != in_total) return false;
    }
    return !job.empty();
  }
};

// ---- member table (host): many streams decoded in one batch (the zip reader) --------------------------------------
// Each member is a raw DEFLATE (method 8) or STORED (method 0) body in[in_off .. in_off + in_len) whose output goes to
// out[out_off .. out_off + out_len), out_len being the size the archive records.  A DEFLATE body of at most one span
// is decoded whole by one thread (decode_span<true, uint8_t>, straight into the output); a larger one runs the
// speculative pipeline above with a Chain of its own, its spans batched with those of the other members in every
// launch.  Each member ends with one status; a bad member never touches another member's output or status.
enum : int32_t { MS_OK = 0, MS_BAD_DATA = 1, MS_WRONG_SIZE = 2, MS_BAD_CRC = 3 };
struct Member {
  uint64_t in_off, in_len, out_off, out_len;
  uint32_t crc32, method;
};
struct FindJob {  // nominal span k >= 1 of the stream in[in_off .. in_off + in_n)
  uint64_t in_off, in_n;
  uint32_t k, pad;
};

struct Batch {
  std::vector<Member> m;
  std::vector<int32_t> status;            // per member
  std::vector<uint32_t> stored;           // members copied as they are
  std::vector<SpanJob> small;             // one decode job per one-span member
  std::vector<uint32_t> large;            // members run through the chain
  std::vector<FindJob> find;              // their nominal spans k >= 1, member by member
  std::vector<uint32_t> find_first;       // large member i's find jobs: find_first[i] .. find_first[i + 1] - 1
  std::vector<Chain> chain;               // per large member
  uint32_t n_rounds = 0;

  // skip (may be null): members already decoded from a seek table, left out of every path here
  void init(const Member *members, uint32_t n, uint64_t span, const uint8_t *skip = nullptr) {
    m.assign(members, members + n);
    status.assign(n, MS_OK);
    stored.clear(); small.clear(); large.clear(); find.clear(); chain.clear();
    find_first.assign(1, 0);
    n_rounds = 0;
    for (uint32_t i = 0; i < n; i++) {
      const Member &x = m[i];
      if (skip && skip[i]) continue;
      if (x.method == 0) {
        if (x.in_len != x.out_len) status[i] = MS_WRONG_SIZE;
        else stored.push_back(i);
      } else if (x.in_len <= span) {
        SpanJob j{key_header(0), KEY_NONE, KEY_NONE, x.out_off, x.out_len, 1, 0, x.in_off, x.in_len, x.out_off, i, 0};
        small.push_back(j);
      } else {
        large.push_back(i);
        const uint32_t n_spans = (uint32_t)((x.in_len + span - 1) / span);
        for (uint32_t k = 1; k < n_spans; k++) find.push_back(FindJob{x.in_off, x.in_len, k, 0});
        find_first.push_back((uint32_t)find.size());
      }
    }
  }
  // cand: the find kernel's result, one key per entry of `find`
  void start_chains(const uint64_t *cand, uint64_t span) {
    chain.assign(large.size(), Chain());
    std::vector<uint64_t> c;
    for (size_t i = 0; i < large.size(); i++) {
      const Member &x = m[large[i]];
      const uint32_t n_spans = find_first[i + 1] - find_first[i] + 1;
      c.assign(n_spans, KEY_NONE);
      for (uint32_t k = 1; k < n_spans; k++) c[k] = cand[find_first[i] + k - 1];
      chain[i].init(c.data(), n_spans, span, x.in_len, GIVE_UP_SPANS, x.in_off, large[i]);
    }
  }
  // the spans of every unfinished chain to count in the next round: jobs[r] is span ref[r].second of chain ref[r].first
  bool pending(std::vector<SpanJob> &jobs, std::vector<std::pair<uint32_t, uint32_t>> &ref) const {
    jobs.clear();
    ref.clear();
    for (uint32_t i = 0; i < chain.size(); i++)
      for (uint32_t s : chain[i].pending()) {
        jobs.push_back(chain[i].job[s]);
        ref.emplace_back(i, s);
      }
    return !jobs.empty();
  }
  void set_results(const std::vector<std::pair<uint32_t, uint32_t>> &ref, const SpanResult *res) {
    n_rounds++;
    std::vector<uint8_t> touched(chain.size(), 0);
    for (size_t r = 0; r < ref.size(); r++) {
      chain[ref[r].first].set_result(ref[r].second, res[r]);
      touched[ref[r].first] = 1;
    }
    for (size_t i = 0; i < chain.size(); i++)
      if (touched[i]) chain[i].advance();
  }
  // After the rounds: the decode jobs of every large member whose chain ended at its recorded size, member by member;
  // first[i] .. first[i + 1] - 1 are the jobs of the i-th of them.  The others get their status here.
  void layout(std::vector<SpanJob> &jobs, std::vector<uint32_t> &first) {
    jobs.clear();
    first.assign(1, 0);
    for (size_t i = 0; i < chain.size(); i++) {
      Chain &c = chain[i];
      const uint32_t mi = large[i];
      if (c.error || !c.done) { status[mi] = MS_BAD_DATA; continue; }
      if (c.layout(m[mi].out_off) != m[mi].out_len) { status[mi] = MS_WRONG_SIZE; continue; }
      jobs.insert(jobs.end(), c.job.begin(), c.job.end());
      first.push_back((uint32_t)jobs.size());
    }
  }
  uint32_t n_spans() const {
    uint32_t s = 0;
    for (const Chain &c : chain) s += (uint32_t)c.job.size();
    return s;
  }
  uint32_t n_rejected() const {
    uint32_t s = 0;
    for (const Chain &c : chain) s += c.n_rejected;
    return s;
  }
  uint32_t n_absorbed() const {
    uint32_t s = 0;
    for (const Chain &c : chain) s += c.n_absorbed;
    return s;
  }
};
// status of a one-span member from its decode
IFL_HD int32_t member_status(int32_t span_status) {
  return span_status == ST_OK ? MS_OK : span_status == ST_OVERFLOW ? MS_WRONG_SIZE : MS_BAD_DATA;
}

}  // namespace ifl
}  // namespace lb2
