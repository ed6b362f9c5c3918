// syms_find_emu.cpp -- TEST HARNESS: runs the PRODUCT's dlsym-style lookup behind lb2_syms_find
// (lambdipy_b200/csrc/elf_syms.cuh: lookup_name with newest = true, found_at) on the CPU, one thread standing in for
// each warp of lb2_syms_find_kernel, over the resolver emulator of syms_emu.cpp (included whole: its index builds the
// arena the lookups read).  It is NOT a CPU fallback: it lives under tests/, is built only by the tests and is never
// loaded by lambdipy_b200/.
#include "syms_emu.cpp"

extern "C" {

// lb2_syms_find: the warp's 32-entry ballot is the first defining entry in scope order; each query's name is read
// from names[name_off ..+ name_len) only (the sanitizer build passes a pool of exactly names_bytes).  -2 (LB2_E_ARG)
// for a query outside the pool or the scope array, or a scope entry that is not an object id.
int lb2emu_syms_find(Emu *s, const Query *queries, uint32_t n, const uint32_t *scope, uint32_t n_scope,
                     const uint8_t *names, uint64_t names_bytes, Found *found) {
  for (uint32_t i = 0; i < n_scope; i++)
    if (scope[i] >= s->objs.size()) return -2;
  for (uint32_t q = 0; q < n; q++)
    if (queries[q].scope_off > n_scope || queries[q].scope_len > n_scope - queries[q].scope_off ||
        queries[q].name_off > names_bytes || queries[q].name_len > names_bytes - queries[q].name_off)
      return -2;
  for (uint32_t q = 0; q < n; q++) {
    const Query &qy = queries[q];
    const uint8_t *name = names + qy.name_off;
    const uint32_t gnu = gnu_hash(name, qy.name_len), sysv = sysv_hash(name, qy.name_len);
    found[q] = Found{NOT_FOUND, 0, 0, 0, 0};
    for (uint32_t e = 0; e < qy.scope_len; e++) {
      const uint32_t id = scope[qy.scope_off + e];
      const Object &d = s->objs[id];
      const int64_t sym = lookup_name(d, (const uint8_t *)d.arena, name, qy.name_len, gnu, sysv, nullptr, nullptr, true);
      if (sym >= 0) {
        found[q] = found_at(id, d, (const uint8_t *)d.arena, (uint32_t)sym);
        break;
      }
    }
  }
  return 0;
}
}

#ifdef LB2EMU_FIND_MAIN
// The sanitizer build (-fsanitize=address,undefined): every file named on the command line is read into a buffer of
// exactly its size and indexed in one batch, and freed; one line per file: status, symbols.  Then each name of
// LB2EMU_FIND (separated by ',') is looked up in the scope of all files, from a pool of exactly the names' bytes; one
// line per name: "find", the object index (-1: none) and the symbol index.
int main(int argc, char **argv) {
  const uint32_t n = argc - 1;
  std::vector<const uint8_t *> ptrs(n + 1);
  std::vector<uint64_t> sizes(n + 1);
  for (uint32_t i = 0; i < n; i++) {
    FILE *f = fopen(argv[i + 1], "rb");
    if (!f) return 3;
    fseek(f, 0, SEEK_END);
    sizes[i] = ftell(f);
    fseek(f, 0, SEEK_SET);
    uint8_t *b = (uint8_t *)malloc(sizes[i] ? sizes[i] : 1);
    if (fread(b, 1, sizes[i], f) != sizes[i]) return 3;
    fclose(f);
    ptrs[i] = b;
  }
  Emu *s = lb2emu_syms_create();
  std::vector<uint32_t> ids(n + 1);
  std::vector<Object> obj(n + 1);
  lb2emu_syms_index(s, ptrs.data(), sizes.data(), n, ids.data(), obj.data());
  for (uint32_t i = 0; i < n; i++) free((void *)ptrs[i]);  // the arena must not need them
  for (uint32_t i = 0; i < n; i++) printf("%d %u\n", obj[i].status, obj[i].nsyms);
  const char *list = getenv("LB2EMU_FIND");
  const uint64_t bytes = list ? strlen(list) : 0;
  uint8_t *pool = (uint8_t *)malloc(bytes ? bytes : 1);
  memcpy(pool, list ? list : "", bytes);
  std::vector<Query> qs;
  for (uint64_t at = 0; list && at <= bytes;) {
    uint64_t e = at;
    while (e < bytes && pool[e] != ',') e++;
    qs.push_back(Query{0, n, (uint32_t)at, (uint32_t)(e - at)});
    at = e + 1;
  }
  std::vector<Found> f(qs.size() + 1);
  if (lb2emu_syms_find(s, qs.data(), (uint32_t)qs.size(), ids.data(), n, pool, bytes, f.data())) return 4;
  for (uint32_t q = 0; q < qs.size(); q++) printf("find %d %u\n", f[q].obj == NOT_FOUND ? -1 : (int)f[q].obj, f[q].sym);
  free(pool);
  lb2emu_syms_destroy(s);
  return 0;
}
#endif
