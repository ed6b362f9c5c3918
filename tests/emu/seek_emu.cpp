// seek_emu.cpp -- TEST HARNESS: runs the PRODUCT's seek-table path (ifl::Table in lambdipy_b200/csrc/inflate_core.cuh)
// on the CPU in the order lb2_inflate_run_table runs it: the table checks, one exact-stop decode per entry into the u16
// arena, Table::accept, the two resolve steps; a refused table falls back to the search pipeline of inflate_emu.cpp.
// It is NOT a CPU fallback: it lives under tests/, is built only by the tests and is never loaded by lambdipy_b200/.
#include "inflate_emu.cpp"

extern "C" {

// entries: n_entries (compressed, decoded) pairs.  *used = 1 when the table was accepted.  Returns what
// lb2emu_inflate returns for the stream.
int lb2emu_table_inflate(const uint8_t *in, uint64_t n, const uint64_t *entries, uint32_t n_entries, uint64_t span_bytes,
                         uint8_t **out, uint64_t *out_n, uint64_t *in_bytes, int *used) {
  *out = nullptr;
  *out_n = 0;
  *used = 0;
  Table t;
  if (t.init(reinterpret_cast<const TableEntry *>(entries), n_entries, n)) {
    std::vector<uint16_t> arena(t.out_total + 1);
    std::vector<SpanResult> res(t.job.size());
    DecodeState *st = new DecodeState;
    for (size_t i = 0; i < t.job.size(); i++) decode_span<true>(in, n, t.job[i], *st, arena.data() + t.job[i].out_off, res[i]);
    delete st;
    if (t.accept(res.data())) {
      *used = 1;
      uint8_t *o = (uint8_t *)malloc(t.out_total + 1);
      int rc = 0;
      for (const SpanJob &j : t.job)
        for (uint64_t i = j.out_len > 32768 ? j.out_len - 32768 : 0; i < j.out_len; i++)
          if (!resolve_value(arena[j.out_off + i], j.out_off, o, o[j.out_off + i])) rc = -100;
      for (const SpanJob &j : t.job)
        for (uint64_t i = 0; i + 32768 < j.out_len; i++)
          if (!resolve_value(arena[j.out_off + i], j.out_off, o, o[j.out_off + i])) rc = -100;
      if (rc) { free(o); return rc; }
      *out = o;
      *out_n = t.out_total;
      *in_bytes = t.in_total;
      return 0;
    }
  }
  uint32_t stats[4];
  return lb2emu_inflate(in, n, span_bytes, out, out_n, stats, in_bytes);
}

}  // extern "C"
