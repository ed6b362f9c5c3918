// parse_emu.cpp -- TEST HARNESS: runs the PRODUCT's optimal-parse core (lambdipy_b200/csrc/deflate_parse.cuh) on the
// CPU the way the best-mode kernel does: Pareto lists from candidates in hash-chain (nearest first) order, the
// forward relaxation one position at a time with its lengths split over 32 lanes, the trace-back, and the tokens
// gathered in order.  It is NOT a CPU fallback: it lives under tests/, is built only by the tests and is never loaded
// by lambdipy_b200/.
#include <vector>

#include "../../lambdipy_b200/csrc/deflate_parse.cuh"

using namespace lb2::dp;

extern "C" {

// cand[cand_off[p] .. cand_off[p + 1]): position p's candidates, length << 16 | (distance - 1), nearest first.
// lists: n * K words, position p's Pareto entries then zeros.
void lb2emu_pareto(const uint32_t *cand, const uint64_t *cand_off, uint32_t n, uint32_t *lists) {
  for (uint32_t p = 0; p < n; p++) {
    uint32_t m = 0, *l = lists + (uint64_t)p * K;
    for (uint64_t c = cand_off[p]; c < cand_off[p + 1]; c++) pareto_insert(l, 1, m, entry_len(cand[c]), entry_dist(cand[c]));
    for (uint32_t k = m; k < K; k++) l[k] = 0;
  }
}

// The cheapest parse of in[0 .. n) over the lists, with the costs lit[256], len[259] (by length) and dist[30] (by
// symbol).  Writes its tokens (the encoder's format) and returns how many; *path_cost gets the path's cost.
uint32_t lb2emu_parse(const uint8_t *in, uint32_t n, const uint32_t *lists, const uint32_t *lit, const uint32_t *len,
                      const uint32_t *dist, uint32_t *tokens, uint64_t *path_cost) {
  Costs c;
  for (int i = 0; i < 256; i++) c.lit[i] = lit[i];
  for (int i = 0; i < 259; i++) c.len[i] = len[i];
  for (int i = 0; i < 30; i++) c.dist[i] = dist[i];
  std::vector<uint16_t> step(n + 1);
  uint32_t ring[RING];
  for (uint32_t s = 0; s < RING; s++) ring[s] = s ? INF : 0u;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t *e = lists + (uint64_t)i * K;
    uint32_t edc[K], m = 0;
    for (uint32_t k = 0; k < K; k++) {
      edc[k] = e[k] ? entry_cost(c, e[k]) : 0u;
      m += e[k] != 0;
    }
    const uint32_t ci = ring[i & (RING - 1)];
    for (uint32_t lane = 0; lane < 32; lane++) relax(i, ci, in[i], e, edc, m, c, ring, step.data(), lane, 32);
    ring[i & (RING - 1)] = INF;
  }
  *path_cost = n ? ring[n & (RING - 1)] : 0;
  trace_back(step.data(), n);
  uint32_t nt = 0;
  for (uint32_t t = 1; t <= n; t++)
    if (step[t] & ON_PATH) {
      const uint32_t l = step[t] & 0x7FFF, s = t - l;
      tokens[nt++] = path_token(l, in[s], lists + (uint64_t)s * K, 1);
    }
  return nt;
}

}  // extern "C"
