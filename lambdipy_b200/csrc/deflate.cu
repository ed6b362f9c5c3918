// deflate.cu -- raw DEFLATE (RFC 1951) encoder and CRC-32 for the gzip and zip writers (lb2_gzip_* / lb2_zip_* in api.cu).
//
// One CTA deflates one chunk of a piece: <= GZ_CHUNK bytes of one segment (a gzip stream's piece or one zip member's
// bytes), described by the chunk table.  It may reference the chunk's `hist` bytes in front of it, which belong to the
// same segment or, for a piece's first segment, to the same stream or file in earlier pieces (the host keeps them in
// front of the piece on the device), so cutting a stream into chunks costs almost nothing in ratio and no match ever
// reaches into another file.  Per chunk:
//   1. in sub-blocks of SUB positions: load the window [pos - 32 KB, sub-block end + 258) into shared memory, build
//      hash chains over it (one warp, __match_any_sync per 32 positions), find each position's longest match among
//      CHAIN candidates (all threads), then walk the sub-block with greedy + one-step lazy parsing (zlib's
//      deflate_slow) on one thread, writing tokens to global memory and counting symbol frequencies;
//   2. build length-limited Huffman codes (15 bits, 7 for the code-length code), price dynamic, fixed and stored
//      coding and keep the smallest;
//   3. pack the tokens: bit offsets from a block-wide exclusive scan of the code lengths, bits ORed into disjoint
//      ranges of a shared-memory buffer (deterministic); close with an empty stored block (Z_SYNC_FLUSH) so the
//      chunk ends byte-aligned, and, if the chunk ends a file, with the final block 03 00.
// In best mode (LB2_DEFLATE_BEST) lb2_deflate_best_kernel then parses every chunk again optimally and rewrites it where
// that is smaller (phases 2 and 3 are shared; the parse itself is in deflate_parse.cuh).
// A second kernel computes per-chunk CRC-32s; a single-CTA kernel scans the chunk sizes and combines the CRCs of each
// segment (GF(2) multiply by x^(8n), as zlib's crc32_combine), and a gather kernel compacts the chunk outputs.
#include "lb2_common.cuh"
#include "copy_device.cuh"
#include "deflate_parse.cuh"

namespace lb2 {
namespace {

constexpr int DF_THREADS = 512;
constexpr int DF_WARPS = DF_THREADS / 32;
constexpr uint32_t SUB = 16384;                         // positions whose matches are found per pass
constexpr uint32_t WIN_CAP = GZ_HIST + SUB + 258;       // bytes one pass looks at
constexpr uint32_t WIN_BYTES = (WIN_CAP + 8 + 15) & ~15u;  // +8: 32-bit reads past the last byte
constexpr uint32_t PREV_BYTES = (WIN_CAP * 2 + 15) & ~15u;
constexpr uint32_t REC_BYTES = SUB * 4;
constexpr uint32_t DF_DYN_SMEM = WIN_BYTES + PREV_BYTES + REC_BYTES;
constexpr int HASH_BITS = 13;
constexpr int CHAIN = 16;        // candidates tried per position
constexpr uint32_t NICE = 128;   // a match this long ends the search
constexpr uint32_t LAZY_MAX = 32;  // matches this long are taken without looking at the next position
constexpr uint32_t TOO_FAR = 4096;  // length-3 matches farther than this cost more than three literals
constexpr uint16_t NIL = 0xFFFF;
constexpr uint32_t OUT_WORDS = GZ_CHUNK_OUT_CAP / 4;
static_assert(OUT_WORDS * 4 <= DF_DYN_SMEM, "packing buffer aliases the match-finding buffers");
static_assert((1u << HASH_BITS) * 2 <= REC_BYTES, "hash heads alias the match records");
static_assert(WIN_CAP < NIL, "window positions are 16-bit");

__constant__ uint16_t c_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                     131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025,
                                     1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

using dp::dext_bits;
using dp::dist_sym;
using dp::len_sym;
using dp::lext_bits;

__device__ __forceinline__ uint32_t hash3(const uint8_t *w, uint32_t i) {
  const uint32_t v = (uint32_t)w[i] | ((uint32_t)w[i + 1] << 8) | ((uint32_t)w[i + 2] << 16);
  return (v * 2654435761u) >> (32 - HASH_BITS);
}
// bytes i..i+3 of the shared-memory window as one little-endian word
__device__ __forceinline__ uint32_t load32(const uint8_t *w, uint32_t i) {
  const uint32_t *p = reinterpret_cast<const uint32_t *>(w) + (i >> 2);
  return __funnelshift_r(p[0], p[1], (i & 3) * 8);
}
__device__ __forceinline__ uint32_t match_len(const uint8_t *w, uint32_t a, uint32_t b, uint32_t max_len) {
  uint32_t l = 0;
  while (l < max_len) {
    const uint32_t x = load32(w, a + l) ^ load32(w, b + l);
    if (x) { l += (__ffs(x) - 1) >> 3; break; }
    l += 4;
  }
  return l < max_len ? l : max_len;
}

struct DfShared {
  uint32_t lfreq[288], dfreq[32], cfreq[20], hfreq[32];
  uint32_t lcode[288], dcode[32], ccode[20];  // bit-reversed code | length << 16
  uint8_t llen[288], dlen[32], clen[20];
  uint16_t sorted[288];
  int A[288];
  int cnt[20];
  uint32_t next_code[20];
  uint8_t rle_sym[320], rle_x[320];
  uint32_t warp_tot[DF_WARPS];
  uint32_t n_rle, hlit, hdist, hclen, hdr_bits, mode, size, ntok, q;
};

// In-place minimum-redundancy code lengths (Moffat & Katajainen) of m >= 2 weights sorted ascending.
__device__ void min_redundancy(int *A, int m) {
  A[0] += A[1];
  int root = 0, leaf = 2, next;
  for (next = 1; next < m - 1; next++) {
    if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; }
    else A[next] = A[leaf++];
    if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; }
    else A[next] += A[leaf++];
  }
  A[m - 2] = 0;
  for (next = m - 3; next >= 0; next--) A[next] = A[A[next]] + 1;
  int avbl = 1, used = 0, dpth = 0;
  root = m - 2;
  next = m - 1;
  while (avbl > 0) {
    while (root >= 0 && A[root] == dpth) { used++; root--; }
    while (avbl > used) { A[next--] = dpth; avbl--; }
    avbl = 2 * used;
    dpth++;
    used = 0;
  }
}

// Code lengths (<= maxbits, complete code) for freq[0..n), n <= 288, at least two non-zero.  Whole block.
__device__ void build_lengths(const uint32_t *freq, int n, int maxbits, uint8_t *len, DfShared &S) {
  const int t = threadIdx.x;
  bool nz = false;
  if (t < n) {
    len[t] = 0;
    const uint32_t f = freq[t];
    if (f) {
      nz = true;
      int r = 0;
      for (int j = 0; j < n; j++) {
        const uint32_t g = freq[j];
        r += (g != 0) & ((g < f) | ((g == f) & (j < t)));
      }
      S.sorted[r] = (uint16_t)t;
    }
  }
  const int m = __syncthreads_count(nz);
  if (t == 0) {
    if (m == 1) {
      len[S.sorted[0]] = 1;
    } else if (m > 1) {
      int *A = S.A;
      for (int k = 0; k < m; k++) A[k] = (int)freq[S.sorted[k]];
      min_redundancy(A, m);
      for (int i = 0; i <= maxbits; i++) S.cnt[i] = 0;
      for (int k = 0; k < m; k++) S.cnt[A[k] < maxbits ? A[k] : maxbits]++;
      uint32_t total = 0;
      for (int i = maxbits; i > 0; i--) total += (uint32_t)S.cnt[i] << (maxbits - i);
      while (total > (1u << maxbits)) {  // clamping over-subscribed the code: lengthen the shortest fitting leaves
        S.cnt[maxbits]--;
        for (int i = maxbits - 1; i > 0; i--)
          if (S.cnt[i]) { S.cnt[i]--; S.cnt[i + 1] += 2; break; }
        total--;
      }
      int j = m;
      for (int i = 1; i <= maxbits; i++)
        for (int l = S.cnt[i]; l > 0; l--) len[S.sorted[--j]] = (uint8_t)i;
    }
  }
  __syncthreads();
}

// Canonical codes (RFC 1951 3.2.2), bit-reversed for LSB-first packing.  Whole block.
__device__ void assign_codes(const uint8_t *len, int n, uint32_t *code, DfShared &S) {
  const int t = threadIdx.x;
  if (t == 0) {
    for (int i = 0; i < 16; i++) S.cnt[i] = 0;
    for (int i = 0; i < n; i++) S.cnt[len[i]]++;
    S.cnt[0] = 0;
    uint32_t c = 0;
    for (int b = 1; b < 16; b++) { c = (c + S.cnt[b - 1]) << 1; S.next_code[b] = c; }
  }
  __syncthreads();
  if (t < n) {
    const uint32_t l = len[t];
    uint32_t c = 0;
    if (l) {
      uint32_t r = 0;
      for (int j = 0; j < t; j++) r += len[j] == l;
      c = (__brev(S.next_code[l] + r) >> (32 - l)) | (l << 16);
    }
    code[t] = c;
  }
  __syncthreads();
}

// Exclusive scan over the block; *total gets the sum.  Whole block.
__device__ uint32_t block_excl_scan(uint32_t v, uint32_t *warp_tot, uint32_t *total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[w] = x;
  __syncthreads();
  if (w == 0) {
    uint32_t s = lane < DF_WARPS ? warp_tot[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < DF_WARPS) warp_tot[lane] = s;
  }
  __syncthreads();
  const uint32_t pre = w ? warp_tot[w - 1] : 0;
  *total = warp_tot[DF_WARPS - 1];
  __syncthreads();
  return pre + x - v;
}

// value v of up to 48 bits at bit offset `off` (LSB first); only non-zero words are touched, so writers of
// neighbouring ranges never race on anything but a commutative OR
__device__ __forceinline__ void or_bits(uint32_t *buf, uint32_t off, uint64_t v) {
  const uint32_t w = off >> 5, sh = off & 31;
  const uint64_t lo = v << sh;
  const uint32_t top = sh ? (uint32_t)(v >> (64 - sh)) : 0u;
  if ((uint32_t)lo) atomicOr(buf + w, (uint32_t)lo);
  if ((uint32_t)(lo >> 32)) atomicOr(buf + w + 1, (uint32_t)(lo >> 32));
  if (top) atomicOr(buf + w + 2, top);
}
// single-thread writer (block header, end of block)
__device__ __forceinline__ void put_bits(uint32_t *buf, uint32_t &pos, uint32_t v, uint32_t n) {
  const uint32_t w = pos >> 5, sh = pos & 31;
  buf[w] |= v << sh;
  if (sh && sh + n > 32) buf[w + 1] |= v >> (32 - sh);
  pos += n;
}

// prev[i]: the nearest earlier position of the window win[0 .. wlen) with the same hash (warp 0; head: the
// 1 << HASH_BITS chain heads, NIL)
__device__ __forceinline__ void build_chains(const uint8_t *win, uint32_t wlen, uint16_t *prev, uint16_t *head) {
  const uint32_t nh = wlen >= 3 ? wlen - 2 : 0;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    for (uint32_t base = 0; base < nh; base += 32) {
      const uint32_t i = base + lane;
      const bool v = i < nh;
      const uint32_t h = v ? hash3(win, i) : 0x80000000u + lane;
      const unsigned grp = __match_any_sync(0xffffffffu, h);
      const unsigned lower = grp & ((1u << lane) - 1);
      uint16_t p = NIL;
      if (lower) p = (uint16_t)(base + 31 - __clz(lower));
      else if (v) p = head[h];
      __syncwarp();
      if (v) {
        prev[i] = p;
        if ((grp >> lane) == 1u) head[h] = (uint16_t)i;
      }
      __syncwarp();
    }
  }
}

// Phase 2: code lengths for S.lfreq / S.dfreq (S.lfreq[256] is set to 1, the end of block) and the cheapest block
// type; S.mode (0 stored, 1 fixed, 2 dynamic) and S.size (bytes, sync flush included, final block not) get the
// choice.  Whole block.
__device__ __forceinline__ void choose_block(DfShared &S, uint32_t clen) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    S.lfreq[256] = 1;  // end of block
    int nz = 0;        // a distance tree needs two codes (one-code trees are incomplete; zlib does the same)
    for (int i = 0; i < 30; i++) { S.hfreq[i] = S.dfreq[i]; nz += S.dfreq[i] != 0; }
    if (nz < 2) { if (!S.hfreq[0]) S.hfreq[0] = 1; else S.hfreq[1] = 1; }
    if (nz == 0) S.hfreq[1] = 1;
  }
  __syncthreads();
  build_lengths(S.lfreq, 286, 15, S.llen, S);
  build_lengths(S.hfreq, 30, 15, S.dlen, S);
  if (tid == 0) {  // code-length sequence with the run-length symbols 16 / 17 / 18
    uint32_t hlit = 286, hdist = 30;
    while (hlit > 257 && S.llen[hlit - 1] == 0) hlit--;
    while (hdist > 1 && S.dlen[hdist - 1] == 0) hdist--;
    for (int i = 0; i < 20; i++) S.cfreq[i] = 0;
    const uint32_t total = hlit + hdist;
    uint32_t nr = 0, i = 0;
    while (i < total) {
      const uint32_t v = i < hlit ? S.llen[i] : S.dlen[i - hlit];
      uint32_t run = 1;
      while (i + run < total && (i + run < hlit ? S.llen[i + run] : S.dlen[i + run - hlit]) == v) run++;
      i += run;
      if (v == 0) {
        while (run >= 11) { const uint32_t r = run < 138 ? run : 138; S.rle_sym[nr] = 18; S.rle_x[nr++] = r - 11; run -= r; }
        if (run >= 3) { S.rle_sym[nr] = 17; S.rle_x[nr++] = run - 3; run = 0; }
      } else {
        S.rle_sym[nr] = v; S.rle_x[nr++] = 0; run--;
        while (run >= 3) { const uint32_t r = run < 6 ? run : 6; S.rle_sym[nr] = 16; S.rle_x[nr++] = r - 3; run -= r; }
      }
      while (run > 0) { S.rle_sym[nr] = v; S.rle_x[nr++] = 0; run--; }
    }
    for (uint32_t k = 0; k < nr; k++) S.cfreq[S.rle_sym[k]]++;
    int nz = 0;
    for (int k = 0; k < 19; k++) nz += S.cfreq[k] != 0;
    if (nz < 2) { if (!S.cfreq[0]) S.cfreq[0] = 1; else S.cfreq[1] = 1; }  // counted below only through rle_sym
    S.n_rle = nr; S.hlit = hlit; S.hdist = hdist;
  }
  __syncthreads();
  build_lengths(S.cfreq, 19, 7, S.clen, S);
  if (tid == 0) {
    uint32_t hclen = 19;
    while (hclen > 4 && S.clen[c_clorder[hclen - 1]] == 0) hclen--;
    uint32_t hdr = 3 + 5 + 5 + 4 + 3 * hclen;
    for (uint32_t k = 0; k < S.n_rle; k++) {
      const uint32_t s = S.rle_sym[k];
      hdr += S.clen[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
    }
    uint32_t dyn = hdr, fix = 3, extra = 0;
    for (int s = 0; s < 286; s++) {
      const uint32_t f = S.lfreq[s];
      dyn += f * S.llen[s];
      fix += f * (s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8);
      extra += f * lext_bits(s);
    }
    for (int s = 0; s < 30; s++) {
      const uint32_t f = S.dfreq[s];
      dyn += f * S.dlen[s];
      fix += f * 5;
      extra += f * dext_bits(s);
    }
    dyn += extra; fix += extra;
    // + the empty stored block: 3 header bits, padding to a byte, LEN / NLEN
    const uint32_t dyn_bytes = (dyn + 3 + 7) / 8 + 4, fix_bytes = (fix + 3 + 7) / 8 + 4;
    const uint32_t stored_bytes = clen + 5 * ((clen + 65534) / 65535) + 5;
    uint32_t mode = 0, size = stored_bytes;
    if (fix_bytes < size) { mode = 1; size = fix_bytes; }
    if (dyn_bytes < size) { mode = 2; size = dyn_bytes; }
    if (clen == 0) size = 0;  // an empty file (stored was cheapest): no blocks, its body is the final block alone
    S.mode = mode; S.size = size; S.hclen = hclen; S.hdr_bits = mode == 2 ? hdr : 3;
  }
  __syncthreads();
}

// Phase 3: chunk c (*ch, clen bytes) in the block type choose_block picked, from its S.ntok tokens at
// a.tokens + ch->start, into its output slot; chunk_size[c] and chunk_mode[c] (| mode_flag) are set.  smem: the
// kernel's dynamic shared memory, used as the packing buffer.  Whole block.
__device__ __forceinline__ void emit_block(const GzPieceArgs &a, const GzChunk *ch, uint32_t c, uint32_t clen,
                                           uint8_t *smem, DfShared &S, uint32_t mode_flag) {
  const int tid = threadIdx.x;
  const uint32_t mode = S.mode, size = S.size;
  // the file ends with this chunk: the final block 03 00 follows its output
  const uint32_t fin = ch->last ? 2 : 0;
  const uint64_t c0 = ch->start;
  uint8_t *out = a.chunk_out + c0 + (uint64_t)c * GZ_OUT_PAD;
  const uint32_t *tok = a.tokens + c0;

  if (mode == 0) {  // stored blocks of <= 65535 bytes, then the empty one
    const uint8_t *in = a.in + c0;
    for (uint32_t i = tid; i < clen; i += DF_THREADS) out[i + 5 * (i / 65535 + 1)] = in[i];
    const uint32_t nblk = (clen + 65534) / 65535;
    if (tid <= (int)nblk) {
      const uint32_t at = tid < (int)nblk ? tid * (65535 + 5) : clen + 5 * nblk;
      const uint32_t len = tid < (int)nblk ? min(65535u, clen - tid * 65535) : 0;
      out[at] = 0;
      out[at + 1] = (uint8_t)len; out[at + 2] = (uint8_t)(len >> 8);
      out[at + 3] = (uint8_t)~len; out[at + 4] = (uint8_t)(~len >> 8);
    }
    if (fin && tid == 0) { out[size] = 0x03; out[size + 1] = 0x00; }
  } else {
    // The fixed literal/length code is the canonical code over all 288 lengths (RFC 1951 3.2.6): the length-8
    // symbols 286 and 287 rank before every length-9 symbol, so leaving them out would shift the codes of the
    // literals 144..255.  A dynamic code has no symbols 286 / 287.
    if (mode == 1) {
      for (int s = tid; s < 288; s += DF_THREADS) S.llen[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
      if (tid < 30) S.dlen[tid] = 5;
    } else if (tid >= 286 && tid < 288) {
      S.llen[tid] = 0;
    }
    __syncthreads();
    assign_codes(S.llen, 288, S.lcode, S);
    assign_codes(S.dlen, 30, S.dcode, S);
    assign_codes(S.clen, 19, S.ccode, S);
    uint32_t *buf = reinterpret_cast<uint32_t *>(smem);
    for (uint32_t i = tid; i < OUT_WORDS; i += DF_THREADS) buf[i] = 0;
    __syncthreads();
    if (tid == 0) {
      uint32_t pos = 0;
      put_bits(buf, pos, mode == 2 ? 4u : 2u, 3);  // BFINAL 0, BTYPE 10 (dynamic) or 01 (fixed)
      if (mode == 2) {
        put_bits(buf, pos, S.hlit - 257, 5);
        put_bits(buf, pos, S.hdist - 1, 5);
        put_bits(buf, pos, S.hclen - 4, 4);
        for (uint32_t k = 0; k < S.hclen; k++) put_bits(buf, pos, S.clen[c_clorder[k]], 3);
        for (uint32_t k = 0; k < S.n_rle; k++) {
          const uint32_t s = S.rle_sym[k], c = S.ccode[s];
          put_bits(buf, pos, c & 0xFFFF, c >> 16);
          if (s >= 16) put_bits(buf, pos, S.rle_x[k], s == 16 ? 2 : s == 17 ? 3 : 7);
        }
      }
    }
    __syncthreads();
    const uint32_t ntok = S.ntok;
    uint32_t bitpos = S.hdr_bits;
    for (uint32_t base = 0; base < ntok; base += DF_THREADS) {
      const uint32_t t = base + tid;
      uint64_t v = 0;
      uint32_t nb = 0;
      if (t < ntok) {
        const uint32_t tk = tok[t];
        if (tk & 0x80000000u) {
          const uint32_t len = ((tk >> 16) & 0xFF) + 3, d0 = tk & 0x7FFF;
          const uint32_t ls = len_sym(len), lc = S.lcode[ls];
          v = lc & 0xFFFF; nb = lc >> 16;
          v |= (uint64_t)(len - c_lbase[ls - 257]) << nb; nb += c_lext[ls - 257];
          const uint32_t ds = dist_sym(d0), dc = S.dcode[ds];
          v |= (uint64_t)(dc & 0xFFFF) << nb; nb += dc >> 16;
          v |= (uint64_t)(d0 + 1 - c_dbase[ds]) << nb; nb += c_dext[ds];
        } else {
          const uint32_t lc = S.lcode[tk];
          v = lc & 0xFFFF; nb = lc >> 16;
        }
      }
      uint32_t total;
      const uint32_t off = bitpos + block_excl_scan(nb, S.warp_tot, &total);
      if (nb) or_bits(buf, off, v);
      bitpos += total;
    }
    __syncthreads();
    if (tid == 0) {
      const uint32_t eob = S.lcode[256];
      put_bits(buf, bitpos, eob & 0xFFFF, eob >> 16);
      const uint32_t nbytes = (bitpos + 3 + 7) / 8;  // empty stored block: 3 zero bits, pad, 00 00 FF FF
      uint8_t *b8 = reinterpret_cast<uint8_t *>(buf);
      b8[nbytes + 2] = 0xFF; b8[nbytes + 3] = 0xFF;
      if (fin) b8[size] = 0x03;  // b8[size + 1] is already 0
    }
    __syncthreads();
    uint32_t *o32 = reinterpret_cast<uint32_t *>(out);
    for (uint32_t i = tid; i < (size + fin + 3) / 4; i += DF_THREADS) o32[i] = buf[i];
  }
  if (tid == 0) {
    a.chunk_size[c] = size + fin;
    a.chunk_mode[c] = clen ? mode | mode_flag : 3;
  }
}

__global__ void __launch_bounds__(DF_THREADS, 1) lb2_deflate_kernel(GzPieceArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t *win = smem;
  uint16_t *prev = reinterpret_cast<uint16_t *>(smem + WIN_BYTES);
  uint32_t *rec = reinterpret_cast<uint32_t *>(smem + WIN_BYTES + PREV_BYTES);
  uint16_t *head = reinterpret_cast<uint16_t *>(rec);  // only while the chains are built
  __shared__ DfShared S;
  const int tid = threadIdx.x;
  // the chunk's fields are read where they are used rather than kept in registers through the match finding
  const GzChunk *ch = a.chunks + blockIdx.x;
  const uint32_t clen = ch->len;

  for (int i = tid; i < 288; i += DF_THREADS) S.lfreq[i] = 0;
  if (tid < 32) S.dfreq[tid] = 0;
  if (tid == 0) S.ntok = 0;

  // ---- 1. match finding and parse, SUB positions per pass ------------------------------------------------
  uint32_t q = 0;
  while (q < clen) {
    const uint32_t hist = ch->hist, back = hist + q < GZ_HIST ? hist + q : GZ_HIST;
    const uint32_t sub_end = q + SUB < clen ? q + SUB : clen;
    const uint32_t we = sub_end + 258 < clen ? sub_end + 258 : clen;  // matches end inside the chunk
    const uint32_t wlen = back + (we - q);
    const uint8_t *src = a.in + ch->start + q - back;
    for (uint32_t i = tid; i < wlen; i += DF_THREADS) win[i] = src[i];
    for (uint32_t i = tid; i < (1u << HASH_BITS); i += DF_THREADS) head[i] = NIL;
    __syncthreads();
    build_chains(win, wlen, prev, head);
    __syncthreads();
    const uint32_t np = sub_end - q;
    for (uint32_t j = tid; j < np; j += DF_THREADS) {
      const uint32_t c = back + j, pos = q + j;
      const uint32_t max_len = clen - pos < 258 ? clen - pos : 258;
      uint32_t best = 0, bdist = 0;
      if (max_len >= 3) {
        uint32_t cand = prev[c];
        for (int k = 0; k < CHAIN && cand != NIL && c - cand <= 32768; k++) {
          if (win[cand + best] == win[c + best]) {
            const uint32_t l = match_len(win, c, cand, max_len);
            if (l > best) {
              best = l;
              bdist = c - cand;
              if (l >= NICE || l >= max_len) break;
            }
          }
          cand = prev[cand];
        }
      }
      if (best < 3 || (best == 3 && bdist > TOO_FAR)) best = 0;
      rec[j] = best | (bdist << 16);
    }
    __syncthreads();
    if (tid == 0) {  // greedy parse with one-step lazy evaluation
      uint32_t *tok = a.tokens + ch->start;
      const uint32_t limit = sub_end < clen ? sub_end - 1 : clen;  // rec[p + 1] must be known
      uint32_t p = q, nt = S.ntok;
      while (p < limit) {
        const uint32_t r = rec[p - q];
        uint32_t l = r & 0x1FF;
        if (l >= 3 && l < LAZY_MAX && p + 1 < clen && (rec[p + 1 - q] & 0x1FF) > l) l = 0;
        if (l >= 3) {
          const uint32_t d = r >> 16;
          tok[nt++] = 0x80000000u | ((l - 3) << 16) | (d - 1);
          S.lfreq[len_sym(l)]++;
          S.dfreq[dist_sym(d - 1)]++;
          p += l;
        } else {
          const uint32_t b = win[back + p - q];
          tok[nt++] = b;
          S.lfreq[b]++;
          p++;
        }
      }
      S.ntok = nt;
      S.q = p;
    }
    __syncthreads();
    q = S.q;
  }

  // ---- 2. codes and the cheapest block type; 3. output ------------------------------------------------------
  choose_block(S, clen);
  emit_block(a, ch, blockIdx.x, clen, smem, S, 0);
}

// ---- best mode (LB2_DEFLATE_BEST): an optimal parse after the greedy one ------------------------------------------
// Runs after lb2_deflate_kernel, whose output every chunk keeps unless the optimal parse is smaller by the same byte
// formula.  One CTA per chunk, chunks claimed from a counter; each CTA owns one workspace slot:
//   1. the greedy tokens' frequencies give the first costs and the size to beat;
//   2. per sub-block as in pass 1, every position's Pareto match list (deflate_parse.cuh) from up to BEST_CHAIN
//      hash-chain candidates, dp::K words per position in the slot;
//   3. BEST_ITERS times: the cheapest path under the current costs (warp 0, one position at a time, its lengths split
//      over the lanes; the lengths of the edges in shared memory), traced back on one thread, its tokens gathered in
//      order by the whole block into the slot; their code (choose_block) prices them and gives the next costs;
//   4. the smallest of these parses, if it beats the greedy one, is written with emit_block.
constexpr uint32_t BEST_CHAIN = 1024;  // hash-chain candidates per position
constexpr uint32_t BEST_ITERS = 4;     // parse -> code -> costs rounds
constexpr uint32_t BEST_UNUSED_BITS = 15;  // cost of a symbol the current code does not have
constexpr uint32_t STEP_OFF = WIN_BYTES;   // u16 step[0 .. GZ_CHUNK] over prev / rec once the match lists are built
constexpr uint32_t PAR_OFF = WIN_BYTES + PREV_BYTES + (1u << HASH_BITS) * 2;  // per-thread Pareto lists, after the heads
static_assert(STEP_OFF + (GZ_CHUNK + 1) * 2 <= DF_DYN_SMEM, "edge lengths fit in the match-finding buffers");
static_assert(PAR_OFF + dp::K * DF_THREADS * 4 <= DF_DYN_SMEM, "Pareto lists fit beside the hash heads");
static_assert(BEST_WS_WORDS == GZ_CHUNK * (dp::K + 1), "slot: match lists, then candidate tokens");

struct BestShared {
  dp::Costs cost;
  uint32_t ring[dp::RING];
  uint32_t ent[32 * dp::K];  // the match lists of 32 positions, staged for warp 0
  uint8_t byte[32];
  uint32_t edc[dp::K];
  uint32_t best_l[288], best_d[32];
  uint32_t best_size, best_ntok, chunk;
};

// next round's costs from the code choose_block just built (the fixed code if it chose that)
__device__ __forceinline__ void set_costs(const DfShared &S, dp::Costs &c) {
  const bool fixed = S.mode == 1;
  for (uint32_t l = threadIdx.x; l < 256 + 259 + 30; l += DF_THREADS) {
    if (l < 256) {
      const uint32_t b = fixed ? (l < 144 ? 8 : 9) : S.llen[l];
      c.lit[l] = b ? b : BEST_UNUSED_BITS;
    } else if (l < 256 + 259) {
      const uint32_t len = l - 256;
      if (len < 3) continue;
      const uint32_t s = len_sym(len);
      const uint32_t b = fixed ? (s < 280 ? 7 : 8) : S.llen[s];
      c.len[len] = (b ? b : BEST_UNUSED_BITS) + lext_bits(s);
    } else {
      const uint32_t s = l - 256 - 259;
      const uint32_t b = fixed ? 5 : S.dlen[s];
      c.dist[s] = (b ? b : BEST_UNUSED_BITS) + dext_bits(s);
    }
  }
}

__global__ void __launch_bounds__(DF_THREADS, 1) lb2_deflate_best_kernel(GzPieceArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t *win = smem;
  uint16_t *prev = reinterpret_cast<uint16_t *>(smem + WIN_BYTES);
  uint16_t *head = reinterpret_cast<uint16_t *>(smem + WIN_BYTES + PREV_BYTES);
  uint32_t *par = reinterpret_cast<uint32_t *>(smem + PAR_OFF);
  uint16_t *step = reinterpret_cast<uint16_t *>(smem + STEP_OFF);
  __shared__ DfShared S;
  __shared__ BestShared B;
  const int tid = threadIdx.x, lane = tid & 31;
  uint32_t *list = a.best_ws + (uint64_t)blockIdx.x * BEST_WS_WORDS;  // dp::K words per position of the chunk
  uint32_t *cand = list + GZ_CHUNK * dp::K;                           // the current round's tokens

  for (;;) {
    __syncthreads();
    if (tid == 0) B.chunk = atomicAdd(a.best_claim, 1u);
    __syncthreads();
    const uint32_t c = B.chunk;
    if (c >= a.n_chunks) return;
    const GzChunk *ch = a.chunks + c;
    const uint32_t clen = ch->len;
    if (clen == 0) continue;
    const uint8_t *in = a.in + ch->start;
    uint32_t *tok = a.tokens + ch->start;

    // ---- 1. the greedy parse: its tokens cover the chunk exactly, those after them are stale -----------------
    for (int i = tid; i < 288; i += DF_THREADS) S.lfreq[i] = 0;
    if (tid < 32) S.dfreq[tid] = 0;
    __syncthreads();
    for (uint32_t base = 0, done = 0; done < clen; base += DF_THREADS) {
      const uint32_t t = base + tid;
      const uint32_t tk = t < clen ? tok[t] : 0;
      const uint32_t len = t < clen ? (tk & 0x80000000u ? ((tk >> 16) & 0xFF) + 3 : 1) : 0;
      uint32_t total;
      const uint32_t at = done + block_excl_scan(len, S.warp_tot, &total);
      if (len && at < clen) {
        if (len == 1) {
          atomicAdd(&S.lfreq[tk], 1u);
        } else {
          atomicAdd(&S.lfreq[len_sym(len)], 1u);
          atomicAdd(&S.dfreq[dist_sym(tk & 0x7FFF)], 1u);
        }
      }
      done += total;
    }
    __syncthreads();
    choose_block(S, clen);
    if (tid == 0) B.best_size = S.size;
    set_costs(S, B.cost);

    // ---- 2. Pareto match lists ----------------------------------------------------------------------------------
    for (uint32_t q = 0; q < clen; q += SUB) {
      const uint32_t hist = ch->hist, back = hist + q < GZ_HIST ? hist + q : GZ_HIST;
      const uint32_t sub_end = q + SUB < clen ? q + SUB : clen;
      const uint32_t we = sub_end + 258 < clen ? sub_end + 258 : clen;
      const uint32_t wlen = back + (we - q);
      const uint8_t *src = in + q - back;
      __syncthreads();
      for (uint32_t i = tid; i < wlen; i += DF_THREADS) win[i] = src[i];
      for (uint32_t i = tid; i < (1u << HASH_BITS); i += DF_THREADS) head[i] = NIL;
      __syncthreads();
      build_chains(win, wlen, prev, head);
      __syncthreads();
      for (uint32_t j = tid; j < sub_end - q; j += DF_THREADS) {
        const uint32_t cp = back + j, pos = q + j;
        const uint32_t max_len = clen - pos < 258 ? clen - pos : 258;
        uint32_t n = 0, best = 2;
        if (max_len >= 3) {
          uint32_t cd = prev[cp];
          for (uint32_t k = 0; k < BEST_CHAIN && cd != NIL && cp - cd <= 32768; k++) {
            if (win[cd + best] == win[cp + best]) {
              const uint32_t l = match_len(win, cp, cd, max_len);
              if (dp::pareto_insert(par + tid, DF_THREADS, n, l, cp - cd)) {
                best = l;
                if (l >= max_len) break;
              }
            }
            cd = prev[cd];
          }
        }
        uint32_t *o = list + (uint64_t)pos * dp::K;
#pragma unroll
        for (uint32_t k = 0; k < dp::K; k++) o[k] = k < n ? par[k * DF_THREADS + tid] : 0u;
      }
    }
    __syncthreads();

    // ---- 3. parse -> code -> costs rounds --------------------------------------------------------------------------
    bool improved = false;
    for (uint32_t it = 0; it < BEST_ITERS; it++) {
      if (tid < 32) {  // the cheapest path: positions in order, the lengths from one position across the lanes
        for (uint32_t s = lane; s < dp::RING; s += 32) B.ring[s] = s ? dp::INF : 0u;
        for (uint32_t i = 0; i < clen; i++) {
          const uint32_t r = i & 31;
          if (r == 0) {  // stage the next 32 positions' lists and bytes
            __syncwarp();
            const uint32_t *src = list + (uint64_t)i * dp::K;
            const uint32_t nw = (clen - i < 32 ? clen - i : 32) * dp::K;
#pragma unroll
            for (uint32_t k = 0; k < dp::K; k++) {
              const uint32_t w = k * 32 + lane;
              B.ent[w] = w < nw ? src[w] : 0u;
            }
            B.byte[lane] = i + lane < clen ? in[i + lane] : 0;
            __syncwarp();
          }
          const uint32_t *e = B.ent + r * dp::K;
          const uint32_t ek = lane < (int)dp::K ? e[lane] : 0u;
          if (lane < (int)dp::K) B.edc[lane] = ek ? dp::entry_cost(B.cost, ek) : 0u;
          const uint32_t n = __popc(__ballot_sync(0xffffffffu, ek != 0));
          __syncwarp();
          const uint32_t ci = B.ring[i & (dp::RING - 1)];
          dp::relax(i, ci, B.byte[r], e, B.edc, n, B.cost, B.ring, step, lane, 32);
          __syncwarp();
          if (lane == 0) B.ring[i & (dp::RING - 1)] = dp::INF;
        }
      }
      __syncthreads();
      if (tid == 0) S.ntok = dp::trace_back(step, clen);
      for (int i = tid; i < 288; i += DF_THREADS) S.lfreq[i] = 0;
      if (tid < 32) S.dfreq[tid] = 0;
      __syncthreads();
      // the path's tokens in order: the marked edge ends, compacted with a block-wide scan
      for (uint32_t base = 0, nt = 0; base < clen; base += DF_THREADS) {
        const uint32_t t = base + 1 + tid;
        const uint32_t sv = t <= clen ? step[t] : 0u;
        const bool on = (sv & dp::ON_PATH) != 0;
        uint32_t total;
        const uint32_t idx = nt + block_excl_scan(on, S.warp_tot, &total);
        if (on) {
          const uint32_t l = sv & 0x7FFF, s = t - l;
          const uint32_t tk = dp::path_token(l, in[s], list + (uint64_t)s * dp::K, 1);
          cand[idx] = tk;
          if (l == 1) {
            atomicAdd(&S.lfreq[tk], 1u);
          } else {
            atomicAdd(&S.lfreq[len_sym(l)], 1u);
            atomicAdd(&S.dfreq[dist_sym(tk & 0x7FFF)], 1u);
          }
        }
        nt += total;
      }
      __syncthreads();
      choose_block(S, clen);
      const bool better = S.size < B.best_size;
      __syncthreads();
      if (better) {  // the smallest round so far: keep its tokens and frequencies
        improved = true;
        for (uint32_t i = tid; i < S.ntok; i += DF_THREADS) tok[i] = cand[i];
        for (int i = tid; i < 288; i += DF_THREADS) B.best_l[i] = S.lfreq[i];
        if (tid < 32) B.best_d[tid] = S.dfreq[tid];
        if (tid == 0) { B.best_size = S.size; B.best_ntok = S.ntok; }
      }
      set_costs(S, B.cost);
      __syncthreads();
    }

    // ---- 4. output ------------------------------------------------------------------------------------------------
    if (improved) {
      for (int i = tid; i < 288; i += DF_THREADS) S.lfreq[i] = B.best_l[i];
      if (tid < 32) S.dfreq[tid] = B.best_d[tid];
      if (tid == 0) S.ntok = B.best_ntok;
      __syncthreads();
      choose_block(S, clen);
      emit_block(a, ch, c, clen, smem, S, GZ_MODE_OPT);
    }
  }
}

// ---- CRC-32 (gzip / zlib polynomial, reflected) ------------------------------------------------------------------
constexpr uint32_t CRC_POLY = 0xedb88320u;
constexpr int CRC_THREADS = 256;
constexpr uint32_t CRC_SUB = GZ_CHUNK / CRC_THREADS;

// a(x) * b(x) mod p(x), both reflected
__device__ uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}
// xt[k] = x^(2^k) mod p
__device__ void init_x2n(uint32_t *xt) {
  uint32_t p = 1u << 30;  // x^1
  xt[0] = p;
  for (int k = 1; k < 32; k++) xt[k] = p = multmodp(p, p);
}
// CRC of A || B from crc(A), crc(B) and len(B)
__device__ uint32_t crc_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b, const uint32_t *xt) {
  uint32_t p = 1u << 31;  // x^0
  uint32_t k = 3;         // x^(8 * len_b) = prod over set bits of len_b of x^(2^(k+3))
  for (uint64_t n = len_b; n; n >>= 1, k++)
    if (n & 1) p = multmodp(xt[k & 31], p);
  return multmodp(p, crc_a) ^ crc_b;
}

// CRC-32 of each chunk of the table (NULL: each GZ_CHUNK-byte chunk of in[0 .. n)); in and every chunk start are
// 16-byte aligned
__global__ void __launch_bounds__(CRC_THREADS) lb2_crc32_kernel(const uint8_t *in, uint64_t n, const GzChunk *chunks,
                                                                uint32_t *chunk_crc) {
  __shared__ uint32_t tab[256], xt[32], s_crc[CRC_THREADS], s_len[CRC_THREADS];
  const int tid = threadIdx.x;
  {
    uint32_t c = tid;
    for (int k = 0; k < 8; k++) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1;
    tab[tid] = c;
  }
  if (tid == 0) init_x2n(xt);
  __syncthreads();
  uint64_t cs;
  uint32_t cl;
  if (chunks) {
    cs = chunks[blockIdx.x].start;
    cl = chunks[blockIdx.x].len;
  } else {
    cs = (uint64_t)blockIdx.x * GZ_CHUNK;
    cl = (uint32_t)(n - cs < GZ_CHUNK ? n - cs : GZ_CHUNK);
  }
  const uint32_t o = (uint32_t)tid * CRC_SUB;
  const uint32_t len = o >= cl ? 0 : (cl - o < CRC_SUB ? cl - o : CRC_SUB);
  const uint8_t *p = in + cs + o;
  uint32_t crc = 0xFFFFFFFFu;
  uint32_t i = 0;
  for (; i + 16 <= len; i += 16) {  // sub-blocks are multiples of 16
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p + i));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 16; k++) crc = tab[(crc ^ (w[k >> 2] >> ((k & 3) * 8))) & 0xFF] ^ (crc >> 8);
  }
  for (; i < len; i++) crc = tab[(crc ^ p[i]) & 0xFF] ^ (crc >> 8);
  s_crc[tid] = len ? ~crc : 0;
  s_len[tid] = len;
  __syncthreads();
  for (int s = 1; s < CRC_THREADS; s <<= 1) {
    if ((tid & (2 * s - 1)) == 0) {
      s_crc[tid] = crc_combine(s_crc[tid], s_crc[tid + s], s_len[tid + s], xt);
      s_len[tid] += s_len[tid + s];
    }
    __syncthreads();
  }
  if (tid == 0) chunk_crc[blockIdx.x] = s_crc[0];
}

// ---- offsets, stream CRC, gather ---------------------------------------------------------------------------------
constexpr int SCAN_THREADS = 1024;

// Offsets of the chunk outputs in `out` and, per segment, its output range and CRC-32.  CRC-32 is linear: crc(c_1 .. c_k) = XOR over i of crc(c_i) * x^(8 L_i), L_i the
// segment bytes after chunk i, so each chunk's term is computed on its own and XORed into its segment.
__global__ void __launch_bounds__(SCAN_THREADS) lb2_gzip_scan_kernel(GzPieceArgs a) {
  __shared__ unsigned long long s_sum[SCAN_THREADS];
  __shared__ uint32_t s_st[SCAN_THREADS], s_fx[SCAN_THREADS], s_op[SCAN_THREADS], xt[32];
  const int tid = threadIdx.x;
  if (tid == 0) init_x2n(xt);
  const uint32_t per_s = (a.n_segs + SCAN_THREADS - 1) / SCAN_THREADS;
  const uint32_t sb = min(a.n_segs, tid * per_s), se = min(a.n_segs, sb + per_s);
  for (uint32_t s = sb; s < se; s++) a.seg_res[s].crc32 = 0;
  __syncthreads();
  const uint32_t per = (a.n_chunks + SCAN_THREADS - 1) / SCAN_THREADS;
  const uint32_t b = min(a.n_chunks, tid * per), e = min(a.n_chunks, b + per);
  unsigned long long sum = 0;
  uint32_t st = 0, fx = 0, op = 0;
  for (uint32_t i = b; i < e; i++) {
    const GzChunk c = a.chunks[i];
    const uint32_t m = a.chunk_mode[i];
    sum += a.chunk_size[i];
    st += (m & 3) == 0;
    fx += (m & 3) == 1;
    op += (m & GZ_MODE_OPT) != 0;
    if (c.len) {
      const GzSeg g = a.segs[c.seg];
      atomicXor(&a.seg_res[c.seg].crc32, crc_combine(a.chunk_crc[i], 0, g.start + g.len - c.start - c.len, xt));
    }
  }
  s_sum[tid] = sum; s_st[tid] = st; s_fx[tid] = fx; s_op[tid] = op;
  __syncthreads();
  for (int o = 1; o < SCAN_THREADS; o <<= 1) {  // inclusive scan of the output bytes
    const unsigned long long y = tid >= o ? s_sum[tid - o] : 0;
    __syncthreads();
    s_sum[tid] += y;
    __syncthreads();
  }
  unsigned long long off = s_sum[tid] - sum;
  for (uint32_t i = b; i < e; i++) { a.chunk_off[i] = off; off += a.chunk_size[i]; }
  for (int s = 1; s < SCAN_THREADS; s <<= 1) {
    if ((tid & (2 * s - 1)) == 0) {
      s_st[tid] += s_st[tid + s];
      s_fx[tid] += s_fx[tid + s];
      s_op[tid] += s_op[tid + s];
    }
    __syncthreads();  // also publishes chunk_off and the XORed segment CRCs to the whole block
  }
  const unsigned long long total = s_sum[SCAN_THREADS - 1];
  const uint32_t state = *a.crc_state;
  for (uint32_t s = sb; s < se; s++) {
    const GzSeg g = a.segs[s];
    uint32_t crc = a.seg_res[s].crc32;
    if (g.flags & GZ_SEG_CONTINUES) crc = crc_combine(state, crc, g.len, xt);
    const unsigned long long o = a.chunk_off[g.first_chunk];
    a.seg_res[s].out_off = o;
    a.seg_res[s].out_len = (s + 1 < a.n_segs ? a.chunk_off[a.segs[s + 1].first_chunk] : total) - o;
    a.seg_res[s].crc32 = crc;
    a.seg_res[s].ended = (g.flags & GZ_SEG_ENDS) != 0;
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t running = a.segs[a.n_segs - 1].flags & GZ_SEG_ENDS ? 0u : a.seg_res[a.n_segs - 1].crc32;
    *a.crc_state = running;
    a.res->crc32 = running;
    a.res->out_bytes = total;
    a.res->n_stored = s_st[0];
    a.res->n_fixed = s_fx[0];
    a.res->n_opt = s_op[0];
  }
}

// CRC-32 of a whole buffer from the per-chunk CRCs of lb2_crc32_kernel
__global__ void __launch_bounds__(SCAN_THREADS) lb2_crc32_combine_kernel(const uint32_t *chunk_crc, uint64_t n, uint32_t *crc) {
  __shared__ unsigned long long s_len[SCAN_THREADS];
  __shared__ uint32_t s_crc[SCAN_THREADS], xt[32];
  const int tid = threadIdx.x;
  if (tid == 0) init_x2n(xt);
  __syncthreads();
  const uint64_t n_chunks = (n + GZ_CHUNK - 1) / GZ_CHUNK;
  const uint64_t per = (n_chunks + SCAN_THREADS - 1) / SCAN_THREADS;
  const uint64_t b = min(n_chunks, tid * per), e = min(n_chunks, b + per);
  uint32_t c = 0;
  unsigned long long len = 0;
  for (uint64_t i = b; i < e; i++) {
    const uint64_t cl = n - i * GZ_CHUNK < GZ_CHUNK ? n - i * GZ_CHUNK : GZ_CHUNK;
    c = crc_combine(c, chunk_crc[i], cl, xt);
    len += cl;
  }
  s_crc[tid] = c;
  s_len[tid] = len;
  __syncthreads();
  for (int s = 1; s < SCAN_THREADS; s <<= 1) {
    if ((tid & (2 * s - 1)) == 0) {
      s_crc[tid] = crc_combine(s_crc[tid], s_crc[tid + s], s_len[tid + s], xt);
      s_len[tid] += s_len[tid + s];
    }
    __syncthreads();
  }
  if (tid == 0) *crc = s_crc[0];
}

// one warp per chunk, with the compaction kernels' byte mover
__global__ void __launch_bounds__(256) lb2_gzip_gather_kernel(GzPieceArgs a) {
  const uint32_t c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= a.n_chunks) return;
  const int lane = threadIdx.x & 31;
  warp_copy_tile(a.chunk_out + a.chunks[c].start + (uint64_t)c * GZ_OUT_PAD, a.out + a.chunk_off[c], a.chunk_size[c], lane);
}

}  // namespace

void launch_deflate(const GzPieceArgs &a, cudaStream_t s) {
  cudaFuncSetAttribute(lb2_deflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_DYN_SMEM);
  lb2_deflate_kernel<<<a.n_chunks, DF_THREADS, DF_DYN_SMEM, s>>>(a);
}
void launch_deflate_best(const GzPieceArgs &a, cudaStream_t s) {
  cudaFuncSetAttribute(lb2_deflate_best_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_DYN_SMEM);
  cudaMemsetAsync(a.best_claim, 0, sizeof(uint32_t), s);
  lb2_deflate_best_kernel<<<a.n_chunks < a.best_slots ? a.n_chunks : a.best_slots, DF_THREADS, DF_DYN_SMEM, s>>>(a);
}
void launch_crc32(const GzPieceArgs &a, cudaStream_t s) {
  lb2_crc32_kernel<<<a.n_chunks, CRC_THREADS, 0, s>>>(a.in, a.n, a.chunks, a.chunk_crc);
}
void launch_crc32(const uint8_t *in, uint64_t n, uint32_t *chunk_crc, uint32_t *crc, cudaStream_t s) {
  if (!n) {
    cudaMemsetAsync(crc, 0, sizeof(uint32_t), s);
    return;
  }
  lb2_crc32_kernel<<<(unsigned)((n + GZ_CHUNK - 1) / GZ_CHUNK), CRC_THREADS, 0, s>>>(in, n, nullptr, chunk_crc);
  lb2_crc32_combine_kernel<<<1, SCAN_THREADS, 0, s>>>(chunk_crc, n, crc);
}
void launch_gzip_compact(const GzPieceArgs &a, cudaStream_t s) {
  lb2_gzip_scan_kernel<<<1, SCAN_THREADS, 0, s>>>(a);
  lb2_gzip_gather_kernel<<<(a.n_chunks + 7) / 8, 256, 0, s>>>(a);
}

}  // namespace lb2
