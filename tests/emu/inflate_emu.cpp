// inflate_emu.cpp -- TEST HARNESS: runs the PRODUCT's inflate core (lambdipy_b200/csrc/inflate_core.cuh) on the CPU
// in the order the CUDA pipeline runs it: candidate search per nominal span, count rounds and the chain, the decode
// pass into the u16 arena, and the two resolve steps.  It lets the CPU suite (-m "not gpu") check the decoder logic
// that ships in the CUDA library against zlib.  It is NOT a CPU fallback: it lives under tests/, is built only by the
// tests and is never loaded by lambdipy_b200/.
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lambdipy_b200/csrc/inflate_core.cuh"

using namespace lb2::ifl;

extern "C" {

// stats: n_spans, n_rounds, n_rejected, n_absorbed.  Returns 0, a span status (< 0) or -100 for a corrupt window.
int lb2emu_inflate(const uint8_t *in, uint64_t n, uint64_t span_bytes, uint8_t **out, uint64_t *out_n, uint32_t *stats,
                   uint64_t *in_bytes) {
  *out = nullptr;
  *out_n = 0;
  const uint32_t n_spans = n > span_bytes ? (uint32_t)((n + span_bytes - 1) / span_bytes) : 1;
  DecodeState *st = new DecodeState;
  std::vector<uint64_t> cand(n_spans, KEY_NONE);
  for (uint32_t k = 1; k < n_spans; k++) {
    const uint64_t end = (uint64_t)(k + 1) * span_bytes < n ? (uint64_t)(k + 1) * span_bytes : n;
    cand[k] = find_candidate(in, n, (uint64_t)k * span_bytes * 8, end * 8, st->hs);
  }
  Chain c;
  c.init(cand.data(), n_spans, span_bytes, n, GIVE_UP_SPANS);
  while (!c.done && !c.error) {
    for (uint32_t i : c.pending()) {
      SpanResult r;
      decode_span<false>(in, n, c.job[i], *st, nullptr, r);
      c.set_result(i, r);
    }
    c.advance();
  }
  stats[0] = (uint32_t)c.job.size();
  stats[1] = c.n_rounds;
  stats[2] = c.n_rejected;
  stats[3] = c.n_absorbed;
  if (c.error) { delete st; return c.error; }
  const uint64_t total = c.layout();
  *in_bytes = c.in_bytes();
  std::vector<uint16_t> arena(total + 1);
  for (const SpanJob &j : c.job) {
    SpanResult r;
    decode_span<true>(in, n, j, *st, arena.data() + j.out_off, r);
    if (r.status) { delete st; return r.status; }
  }
  delete st;
  uint8_t *o = (uint8_t *)malloc(total + 1);
  int rc = 0;
  for (const SpanJob &j : c.job)  // the window of every span: its last 32 KB, in span order
    for (uint64_t i = j.out_len > 32768 ? j.out_len - 32768 : 0; i < j.out_len; i++)
      if (!resolve_value(arena[j.out_off + i], j.out_off, o, o[j.out_off + i])) rc = -100;
  for (const SpanJob &j : c.job)  // everything else
    for (uint64_t i = 0; i + 32768 < j.out_len; i++)
      if (!resolve_value(arena[j.out_off + i], j.out_off, o, o[j.out_off + i])) rc = -100;
  if (rc) { free(o); return rc; }
  *out = o;
  *out_n = total;
  return 0;
}

// Keys of the dynamic and stored blocks a serial decode from bit 0 passes through (the first block is not listed).
// Returns how many were found (at most cap are written), or a span status (< 0).
int64_t lb2emu_block_keys(const uint8_t *in, uint64_t n, uint64_t *keys, uint64_t cap) {
  DecodeState *st = new DecodeState;
  SpanJob j{key_header(0), 0, KEY_NONE, 0, 0, 1, 0};
  int64_t count = 0;
  for (;;) {
    SpanResult r;
    decode_span<false>(in, n, j, *st, nullptr, r);
    if (r.status) { count = r.status; break; }
    if (r.final) break;
    if ((uint64_t)count < cap) keys[count] = r.end_key;
    count++;
    j.start_key = r.end_key;
    j.first = 0;
  }
  delete st;
  return count;
}

// the candidate filter at bit p: a key, or ~0
uint64_t lb2emu_candidate(const uint8_t *in, uint64_t n, uint64_t p) {
  HdrScratch *s = new HdrScratch;
  const uint64_t k = candidate_at(in, n, p, *s);
  delete s;
  return k;
}

void lb2emu_free(void *p) { free(p); }

}  // extern "C"
