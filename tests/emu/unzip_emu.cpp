// unzip_emu.cpp -- TEST HARNESS: runs the PRODUCT's member-table pipeline (ifl::Batch and the decoding core of
// lambdipy_b200/csrc/inflate_core.cuh) on the CPU in the order lb2_unzip_run runs it on the GPU: STORED copies, the
// one-span members decoded whole as bytes, then for the larger members the candidate search per (member, nominal
// span), count rounds over every unfinished chain, the decode pass into the u16 arena at each member's offset, the
// per-member window walk and the per-span resolve.  CRC-32 is left to the caller.  It is NOT a CPU fallback: it lives
// under tests/, is built only by the tests and is never loaded by lambdipy_b200/.
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lambdipy_b200/csrc/inflate_core.cuh"

using namespace lb2::ifl;

extern "C" {

// members: n_members rows of (body_off, body_len, size, method).  Fills out_off[i] and status[i] (MS_*, CRC not
// checked); *out receives the output buffer (free with lb2emu_free), *out_n its size.  stats: n_stored, n_small,
// n_large, n_spans, n_rounds, n_rejected.
int lb2emu_unzip(const uint8_t *in, uint64_t n, const uint64_t *rows, uint32_t n_members, uint64_t span, uint8_t **out,
                 uint64_t *out_n, uint64_t *out_off, int32_t *status, uint32_t *stats) {
  std::vector<Member> m(n_members);
  uint64_t total = 0;
  for (uint32_t i = 0; i < n_members; i++) {
    const uint64_t *r = rows + 4 * i;
    m[i] = Member{r[0], r[1], total, r[2], 0, (uint32_t)r[3]};
    total = (total + r[2] + 15) & ~15ull;
  }
  Batch b;
  b.init(m.data(), n_members, span);
  uint8_t *o = (uint8_t *)calloc(total + 1, 1);
  std::vector<int32_t> dev(n_members, MS_OK);
  DecodeState *st = new DecodeState;
  for (uint32_t i : b.stored) memcpy(o + m[i].out_off, in + m[i].in_off, m[i].out_len);
  for (const SpanJob &j : b.small) {
    SpanResult r;
    decode_span<true, uint8_t>(in + j.in_off, j.in_n, j, *st, o + j.out_off, r);
    dev[j.member] = member_status(r.status);
  }
  std::vector<uint64_t> cand(b.find.size());
  for (size_t f = 0; f < b.find.size(); f++) {
    const FindJob &fj = b.find[f];
    const uint64_t end = (fj.k + 1) * span < fj.in_n ? (fj.k + 1) * span : fj.in_n;
    cand[f] = find_candidate(in + fj.in_off, fj.in_n, fj.k * span * 8, end * 8, st->hs);
  }
  b.start_chains(cand.data(), span);
  std::vector<SpanJob> jobs;
  std::vector<std::pair<uint32_t, uint32_t>> ref;
  std::vector<SpanResult> res;
  while (b.pending(jobs, ref)) {
    res.resize(jobs.size());
    for (size_t i = 0; i < jobs.size(); i++)
      decode_span<false>(in + jobs[i].in_off, jobs[i].in_n, jobs[i], *st, (uint16_t *)nullptr, res[i]);
    b.set_results(ref, res.data());
  }
  stats[0] = (uint32_t)b.stored.size();
  stats[1] = (uint32_t)b.small.size();
  stats[2] = (uint32_t)b.large.size();
  stats[4] = b.n_rounds;
  stats[5] = b.n_rejected();
  std::vector<uint32_t> first;
  b.layout(jobs, first);
  stats[3] = (uint32_t)jobs.size();
  std::vector<uint16_t> arena(total + 1);
  for (const SpanJob &j : jobs) {
    SpanResult r;
    decode_span<true>(in + j.in_off, j.in_n, j, *st, arena.data() + j.out_off, r);
    if (r.status) dev[j.member] = r.status;
  }
  delete st;
  for (size_t s = 0; s + 1 < first.size(); s++)  // window: one walk per member, its spans in order
    for (uint32_t k = first[s]; k < first[s + 1]; k++) {
      const SpanJob &j = jobs[k];
      for (uint64_t i = j.out_len > 32768 ? j.out_len - 32768 : 0; i < j.out_len; i++)
        if (!resolve_value(arena[j.out_off + i], j.out_off, o, o[j.out_off + i], j.out_base)) dev[j.member] = -100;
    }
  for (const SpanJob &j : jobs)  // everything else
    for (uint64_t i = 0; i + 32768 < j.out_len; i++)
      if (!resolve_value(arena[j.out_off + i], j.out_off, o, o[j.out_off + i], j.out_base)) dev[j.member] = -100;
  for (uint32_t i = 0; i < n_members; i++) {
    out_off[i] = m[i].out_off;
    status[i] = b.status[i] != MS_OK ? b.status[i] : dev[i] < 0 ? (int32_t)MS_BAD_DATA : dev[i];
  }
  *out = o;
  *out_n = total;
  return 0;
}

void lb2emu_free(void *p) { free(p); }

}  // extern "C"
