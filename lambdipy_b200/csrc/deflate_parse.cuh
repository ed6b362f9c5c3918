// deflate_parse.cuh -- the per-chunk optimal parse of the thorough DEFLATE mode (LB2_DEFLATE_BEST), shared by the
// best-mode kernel (deflate.cu) and the CPU harness of the tests (tests/emu/parse_emu.cpp).
//
// A chunk of n bytes is a graph on positions 0..n: a literal edge i -> i + 1, and for every match the match finder
// keeps at i, an edge i -> i + l for each length l it covers.  Edge weights are bit costs under a Huffman code; the
// cheapest path from 0 to n is the parse.  Positions are visited in order, so the costs of the 259 positions an edge
// can reach are all that is kept (a ring), plus, per position, the length of the edge the cheapest path arrives by.
//
// Matches.  At each position the finder walks the hash chain nearest first and keeps the Pareto set: a candidate
// joins only if it is longer than every nearer one, so the set is ascending in length and distance.  Entry k covers
// the lengths (length of entry k - 1) + 1 .. its own length (entry 0 from 3) at its own distance, the nearest
// distance that reaches them.  With K entries held, a longer candidate drops the shortest.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define DP_HD __host__ __device__ __forceinline__
#else
#define DP_HD inline
#endif

namespace lb2 {
namespace dp {

constexpr uint32_t K = 8;               // Pareto entries kept per position
constexpr uint32_t RING = 512;          // path costs in flight: a power of two > 258
constexpr uint32_t INF = 0xFFFFFFFFu;
constexpr uint16_t ON_PATH = 0x8000;    // step[t]: the edge into t is on the traced path

// ---- DEFLATE symbols (RFC 1951 3.2.5) ---------------------------------------------------------------------------
DP_HD uint32_t log2_floor(uint32_t v) {
#ifdef __CUDA_ARCH__
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}
DP_HD uint32_t len_sym(uint32_t len) {  // 3..258 -> 257..285
  if (len == 258) return 285;
  const uint32_t l = len - 3;
  if (l < 8) return 257 + l;
  const uint32_t n = log2_floor(l);
  return 257 + 4 * (n - 1) + ((l >> (n - 2)) & 3);
}
DP_HD uint32_t dist_sym(uint32_t d0) {  // distance - 1 -> 0..29
  if (d0 < 4) return d0;
  const uint32_t n = log2_floor(d0);
  return 2 * n + ((d0 >> (n - 1)) & 1);
}
DP_HD uint32_t lext_bits(uint32_t sym) { return sym >= 265 && sym < 285 ? (sym - 261) / 4 : 0; }
DP_HD uint32_t dext_bits(uint32_t sym) { return sym >= 4 ? sym / 2 - 1 : 0; }

// the encoder's token: a literal byte, or 0x80000000 | (length - 3) << 16 | (distance - 1)
DP_HD uint32_t match_token(uint32_t len, uint32_t dist) { return 0x80000000u | ((len - 3) << 16) | (dist - 1); }

// ---- Pareto match lists: entry = length << 16 | (distance - 1), 0 = none ------------------------------------------
DP_HD uint32_t entry_len(uint32_t e) { return e >> 16; }
DP_HD uint32_t entry_dist(uint32_t e) { return (e & 0xFFFF) + 1; }

// Offer the candidate (len, dist) to the list[k * stride], k < n, of one position; candidates come in increasing
// distance.  Returns whether it joined.
DP_HD bool pareto_insert(uint32_t *list, uint32_t stride, uint32_t &n, uint32_t len, uint32_t dist) {
  if (len <= (n ? entry_len(list[(n - 1) * stride]) : 2u)) return false;
  if (n == K) {  // keep the longest
    for (uint32_t k = 0; k + 1 < K; k++) list[k * stride] = list[(k + 1) * stride];
    n--;
  }
  list[n++ * stride] = (len << 16) | (dist - 1);
  return true;
}

// ---- costs -----------------------------------------------------------------------------------------------------
// Bits of every literal, of every match length (symbol + extra bits) and of every distance symbol (+ extra bits).
struct Costs {
  uint32_t lit[256];
  uint32_t len[259];
  uint32_t dist[30];
};
DP_HD uint32_t entry_cost(const Costs &c, uint32_t e) { return c.dist[dist_sym(e & 0xFFFF)]; }

// ---- relaxation ----------------------------------------------------------------------------------------------------
// The edges leaving position i, whose cheapest path costs ci: the literal `byte` (lane 0), and every match length 3 ..
// length of e[n - 1] at the distance of the first entry that reaches it (edc[k]: entry_cost of e[k]).  Lane `lane` of
// `lanes` takes the lengths 3 + lane, 3 + lane + lanes, ...  The targets of one position are distinct, so lanes never
// write the same ring slot.  Only a strictly smaller cost replaces a target's, so of several cheapest paths the one
// whose last edge leaves the earliest position (and, from one position, the shorter literal) is kept: the parse is
// the same however the lanes are scheduled.  step[t] gets the length of the edge into t (1: the literal).
DP_HD void relax(uint32_t i, uint32_t ci, uint32_t byte, const uint32_t *e, const uint32_t *edc, uint32_t n,
                 const Costs &c, uint32_t *ring, uint16_t *step, uint32_t lane, uint32_t lanes) {
  if (lane == 0) {
    const uint32_t v = ci + c.lit[byte];
    uint32_t &r = ring[(i + 1) & (RING - 1)];
    if (v < r) { r = v; step[i + 1] = 1; }
  }
  const uint32_t maxl = n ? entry_len(e[n - 1]) : 0;
  uint32_t k = 0;
  for (uint32_t l = 3 + lane; l <= maxl; l += lanes) {
    while (entry_len(e[k]) < l) k++;
    const uint32_t v = ci + c.len[l] + edc[k];
    uint32_t &r = ring[(i + l) & (RING - 1)];
    if (v < r) { r = v; step[i + l] = (uint16_t)l; }
  }
}

// ---- trace-back -------------------------------------------------------------------------------------------------------
// Mark the edges of the cheapest path into n (ON_PATH on step[t] of each edge's end t); returns how many there are.
DP_HD uint32_t trace_back(uint16_t *step, uint32_t n) {
  uint32_t m = 0;
  for (uint32_t t = n; t > 0; m++) {
    const uint32_t l = step[t];
    step[t] = (uint16_t)(l | ON_PATH);
    t -= l;
  }
  return m;
}
// The token of the marked edge of length l that ends at t: a literal, or the match from s = t - l at the distance of
// the first of the entries e[k * stride] at s that reaches l -- the edge relax() priced.
DP_HD uint32_t path_token(uint32_t l, uint32_t byte_at_s, const uint32_t *e, uint32_t stride) {
  if (l == 1) return byte_at_s;
  uint32_t k = 0;
  while (entry_len(e[k * stride]) < l) k++;
  return match_token(l, entry_dist(e[k * stride]));
}

}  // namespace dp
}  // namespace lb2
