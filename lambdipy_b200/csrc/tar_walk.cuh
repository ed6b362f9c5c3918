// tar_walk.cuh -- the member walk of a tar stream behind lb2_tar_index (kernel in tar.cu), shared with the CPU emulator
// of the tests (tests/emu/tar_emu.cpp).
//
// It restates how Python 3.12's tarfile lists members (TarFile.next, TarInfo.frombuf, _proc_member and the _proc_*
// methods) for USTAR, GNU, PAX and v7 headers, only far enough to know which bytes that listing reads: every header
// block, the byte in front of it (TarFile.next reads offset - 1 to check that the previous member's data exists), the
// data of GNU long-name / long-link and pax headers, GNU old-sparse extension blocks and the first data block of a pax
// 1.0 sparse member.  The caller still lists the members with tarfile itself, from those bytes; the walk only saves it
// from fetching them one by one.  Where the walk is unsure it stops (STOP_UNSUPPORTED) and the caller fetches the rest.
//
// Rules restated from tarfile:
//   * data is skipped, rounded up to 512, only for isreg() types and types outside SUPPORTED_TYPES -- not for
//     directories or links, whatever their size field says;
//   * numbers are `nti`: base-256 after a 0x80 / 0xFF byte, else octal up to the first NUL, blanks stripped;
//   * the checksum matches tarfile's unsigned or signed sum, the checksum field counted as spaces;
//   * an `x` (or Solaris `X`) header's `size` record replaces the size of the member it precedes (the first such
//     header in front of the member wins, as in the nested _proc_pax calls); `g` headers do not move the walk;
//   * an AREGTYPE header whose name ends in '/' is a directory, except right after an extended header (dircheck);
//   * the walk stops at an all-zero block, a header tarfile refuses, or the end of the data, and gathers that block.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define TW_HD __host__ __device__ __forceinline__
#else
#define TW_HD inline
#endif

namespace lb2 {
namespace tarw {

constexpr uint64_t BLOCK = 512;
constexpr uint64_t EXT_CAP = 1ull << 20;  // GNU long names and pax records gathered per header, at most

// why the walk stopped (LB2_TAR_STOP_* in lambdipy_b200.h)
enum : uint32_t { STOP_ZERO = 1, STOP_BAD_HEADER = 2, STOP_END = 3, STOP_UNSUPPORTED = 4 };

struct Range {
  uint64_t off, len;
};

struct WalkResult {
  uint64_t members;   // member headers walked (extended headers not counted)
  uint64_t stop_off;  // the offset of the block the walk stopped at
  uint32_t reason;    // STOP_*
};

TW_HD uint64_t round_block(uint64_t x) { return (x + BLOCK - 1) & ~(BLOCK - 1); }

TW_HD bool is_blank(uint8_t c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x1f); }

// tarfile.nti over s[0 .. len): false where tarfile raises InvalidHeaderError (or the value does not fit in 63 bits)
TW_HD bool nti(const uint8_t *s, int len, int64_t &v) {
  if (s[0] == 0x80 || s[0] == 0xFF) {
    const uint8_t sign = s[0] == 0xFF ? 0xFF : 0;
    uint64_t x = 0;
    for (int i = 1; i < len; i++) {
      if (i < len - 8 && s[i] != sign) return false;
      x = x << 8 | s[i];
    }
    v = (int64_t)x;
    return sign ? v < 0 : v >= 0;
  }
  int e = 0;
  while (e < len && s[e]) e++;
  for (int i = 0; i < e; i++)
    if (s[i] >= 0x80) return false;
  int b = 0;
  while (b < e && is_blank(s[b])) b++;
  while (e > b && is_blank(s[e - 1])) e--;
  v = 0;
  if (b == e) return true;
  const bool neg = s[b] == '-';
  if (s[b] == '-' || s[b] == '+') b++;
  if (b == e) return false;
  uint64_t x = 0;
  for (; b < e; b++) {
    if (s[b] < '0' || s[b] > '7' || (x >> 59)) return false;
    x = x * 8 + (s[b] - '0');
  }
  v = neg ? -(int64_t)x : (int64_t)x;
  return true;
}

// the name field (up to its first NUL) ends in '/'
TW_HD bool name_ends_slash(const uint8_t *h) {
  int e = 0;
  while (e < 100 && h[e]) e++;
  return e > 0 && h[e - 1] == '/';
}

TW_HD bool key_is(const uint8_t *k, uint64_t n, const char *want) {
  uint64_t i = 0;
  for (; want[i]; i++)
    if (i >= n || k[i] != (uint8_t)want[i]) return false;
  return i == n;
}

struct PaxInfo {
  int64_t size = -1;          // the last `size` record
  bool sparse_size = false;   // GNU.sparse.size / realsize: they set the size too
  bool major1 = false, minor0 = false;  // GNU.sparse.major=1, GNU.sparse.minor=0: a 1.0 sparse map leads the data
};

// The records of a pax header, framed as _proc_pax frames them over buf[0 .. len) (the data rounded up to 512); false
// where tarfile raises, or a `size` value is not plain decimal.
TW_HD bool pax_scan(const uint8_t *buf, uint64_t len, PaxInfo &p) {
  uint64_t pos = 0;
  while (pos < len && buf[pos] != 0) {
    uint64_t q = pos, length = 0;
    while (q < len && q - pos < 20 && buf[q] >= '0' && buf[q] <= '9') length = length * 10 + (buf[q++] - '0');
    if (q == pos || q >= len || buf[q] != ' ') return false;
    if (length < 5 || length > len - pos) return false;
    const uint64_t last = pos + length - 1;  // the record's '\n'
    const uint64_t k0 = q + 1;
    if (k0 > last) return false;
    uint64_t eq = k0;
    while (eq < last && buf[eq] != '=') eq++;
    if (eq == k0 || eq >= last || buf[last] != '\n') return false;
    const uint8_t *key = buf + k0, *val = buf + eq + 1;
    const uint64_t kn = eq - k0, vn = last - eq - 1;
    if (key_is(key, kn, "size")) {
      if (vn == 0 || vn > 18) return false;
      int64_t x = 0;
      for (uint64_t i = 0; i < vn; i++) {
        if (val[i] < '0' || val[i] > '9') return false;
        x = x * 10 + (val[i] - '0');
      }
      p.size = x;
    } else if (key_is(key, kn, "GNU.sparse.size") || key_is(key, kn, "GNU.sparse.realsize")) {
      p.sparse_size = true;
    } else if (key_is(key, kn, "GNU.sparse.major")) {
      p.major1 = vn == 1 && val[0] == '1';
    } else if (key_is(key, kn, "GNU.sparse.minor")) {
      p.minor0 = vn == 1 && val[0] == '0';
    }
    pos += length;
  }
  return true;
}

// The walk.  Io supplies, for the kernel one warp and for the emulator one thread:
//   load(off)          the block at off (off + 512 <= n) into io.h, with io.su / io.ss (tarfile's unsigned and signed
//                      checksums) and io.zero (all 512 bytes zero);
//   gather(off, len)   records [off, off + len) as a range tarfile reads, with its bytes.
// Every lane of the warp runs the same walk on the same values.
template <class Io> TW_HD void walk(Io &io, const uint8_t *tar, uint64_t n, WalkResult &r) {
  uint64_t off = 0, members = 0;
  int64_t pax_size = -1;  // the size record of the first `x` header in front of the member
  bool chain = false;     // the block at off follows an extended header (read without a seek, no dircheck)
  bool sparse10 = false;
  uint32_t why = 0;
  for (;;) {
    if (!chain && off > 0) {
      if (off - 1 >= n) { why = STOP_END; break; }
      io.gather(off - 1, 1);
    }
    if (off >= n) { why = STOP_END; break; }
    if (n - off < BLOCK) { io.gather(off, n - off); why = STOP_END; break; }
    io.load(off);
    io.gather(off, BLOCK);
    if (io.zero) { why = STOP_ZERO; break; }
    const uint8_t *h = io.h;
    int64_t chk, size, v;
    if (!nti(h + 148, 8, chk) || (chk != io.su && chk != io.ss)) { why = STOP_BAD_HEADER; break; }
    if (!nti(h + 100, 8, v) || !nti(h + 108, 8, v) || !nti(h + 116, 8, v) || !nti(h + 124, 12, size) ||
        !nti(h + 136, 12, v) || !nti(h + 329, 8, v) || !nti(h + 337, 8, v)) { why = STOP_BAD_HEADER; break; }
    const uint8_t t = h[156];
    uint64_t data = off + BLOCK;
    if (t == 'L' || t == 'K' || t == 'x' || t == 'X' || t == 'g') {
      if (size < 0 || (uint64_t)size > EXT_CAP) { why = STOP_UNSUPPORTED; break; }
      const uint64_t len = round_block((uint64_t)size), have = len < n - data ? len : n - data;
      if (have) io.gather(data, have);
      if (t != 'L' && t != 'K') {
        PaxInfo p;
        if (!pax_scan(tar + data, have, p)) { why = STOP_UNSUPPORTED; break; }
        if (t == 'g') {
          if (p.size >= 0 || p.sparse_size) { why = STOP_UNSUPPORTED; break; }  // a global size: not followed here
        } else {
          if (p.size >= 0 && p.sparse_size) { why = STOP_UNSUPPORTED; break; }
          if (pax_size < 0) pax_size = p.size;
          sparse10 = sparse10 || (p.major1 && p.minor0);
        }
      }
      off = data + len;
      chain = true;
      continue;
    }
    members++;
    const bool dir = t == '5' || (t == 0 && !chain && name_ends_slash(h));
    const bool reg = !dir && (t == '0' || t == 0 || t == '7' || t == 'S');
    const bool supported = dir || reg || (t >= '1' && t <= '6');
    if (t == 'S') {  // old GNU sparse: extension blocks follow the header while the previous one says so
      bool ext = h[482] != 0;
      while (ext) {
        if (n - data < BLOCK) { io.gather(data, n - data); why = STOP_END; break; }
        io.load(data);
        io.gather(data, BLOCK);
        ext = io.h[504] != 0;
        data += BLOCK;
      }
      if (why) break;
    }
    if (sparse10 && data < n) io.gather(data, n - data < BLOCK ? n - data : BLOCK);
    const int64_t sz = pax_size >= 0 ? pax_size : size;
    if (reg || !supported) {
      if (sz < 0) { why = STOP_BAD_HEADER; break; }
      data += round_block((uint64_t)sz);
    }
    off = data;
    pax_size = -1;
    sparse10 = chain = false;
  }
  r.members = members;
  r.stop_off = off;
  r.reason = why;
}

}  // namespace tarw
}  // namespace lb2
