/*
 * lambdipy_b200.h -- C ABI of the H100 (sm_90a) ELF strip library, liblambdipy_b200.so.
 *
 * What it replaces.  The reference (customink/lambdipy) has no FFI for this step: it strips the
 * build tree by running one shell line inside a generated script,
 *
 *     find {install_dir}/ -name "*.so" | xargs strip        /root/reference/lambdipy/project_build.py:260
 *
 * executed by install_non_resolved_requirements() (project_build.py:234-277; Popen at :268, docker
 * exec at :274) before the script is removed (:277).  The entry points below are what a ctypes
 * binding placed at that spot calls instead (see INTEGRATION.md for the reference-side stub):
 *
 *   lb2_strip_tree()          == the whole shell line: select basename "*.so" under a root
 *                                (find, :260), strip each regular ELF in place (strip, :260) the way
 *                                GNU strip 2.42 does: new contents written into the EXISTING inode
 *                                (mode, owner and other hard links kept; mtime not).
 *   lb2_strip_host()          == `strip` over a batch of files already read into host memory
 *                                (what xargs hands to one strip process), results to host memory.
 *   lb2_strip_device_async()  == the same batch with input and output arenas resident in HBM
 *                                (benchmark / pipeline building block; with lb2_unzip_device_output in front
 *                                and lb2_zip_submit_device behind it, the same line applied to the "*.so"
 *                                members of a zip without unpacking it).
 *
 * Result contract: for every file with status LB2_ST_OK the output bytes are identical to
 * `strip --strip-unneeded -o OUT IN` of GNU Binutils 2.42 (== flagless `strip` for ET_DYN/ET_EXEC).
 * Files the device planner does not cover get a positive status and no output; lb2_strip_tree can
 * hand exactly those to the host `strip` binary (LB2_TREE_FALLBACK_HOST_STRIP) so the tree ends up
 * identical to the reference's, and reports how many took that route.
 *
 * Conventions: plain C types; the caller owns every buffer it passes; the library keeps no pointer
 * past a call except where stated (async call: until lb2_batch_results); functions return 0 on
 * success or a negative LB2_E_* code and never throw; one context per thread and device.
 * There is no CPU implementation behind this ABI: without a CUDA device lb2_ctx_create fails.
 */
#ifndef LAMBDIPY_B200_H
#define LAMBDIPY_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct lb2_ctx lb2_ctx;

/* library return codes */
enum {
  LB2_OK = 0,
  LB2_E_CUDA = -1,        /* CUDA runtime error; text in lb2_last_error */
  LB2_E_ARG = -2,         /* bad argument (NULL, unaligned offsets, ...) */
  LB2_E_CAPACITY = -3,    /* output arena too small (stats.out_bytes_needed says how much); lb2_inflate_run: the
                             stream does not fit in device memory */
  LB2_E_IO = -4,          /* filesystem error in lb2_strip_tree */
  LB2_E_NODEVICE = -5,    /* no usable CUDA device */
  LB2_E_STATE = -6,       /* call out of order (no batch in flight, ...) */
  LB2_E_DATA = -7         /* lb2_inflate_run: the DEFLATE stream is invalid or truncated */
};

/* per-file status written by the plan kernel */
enum {
  LB2_ST_OK = 0,
  LB2_ST_NOT_ELF = 1,            /* GNU strip: "file format not recognized" */
  LB2_ST_NOT_ELF64LE = 2,
  LB2_ST_BAD_TYPE = 3,           /* ET_REL, ET_CORE ... */
  LB2_ST_NO_SECTIONS = 4,        /* GNU strip: "has no sections" */
  LB2_ST_XINDEX = 5,
  LB2_ST_UNSUPPORTED_LAYOUT = 6, /* a layout rule the planner does not implement */
  LB2_ST_BAD_NOTES = 7,          /* corrupt .gnu.build.attributes (objcopy refuses too) */
  LB2_ST_PLANNER_LIMIT = 8,      /* > 64 sections, > 32 phdrs, > 2 KB of section names, > 8 KB notes */
  LB2_ST_MALFORMED = -1
};

/* flags for the strip calls */
#define LB2_F_NO_MERGE_NOTES 1u /* behave like `strip --no-merge-notes` */

/* flags for lb2_strip_tree */
#define LB2_TREE_FALLBACK_HOST_STRIP 0x100u /* unsupported ELF files: run the host `strip` on them  */
#define LB2_TREE_TOLERATE_NON_ELF    0x200u /* non-ELF "*.so": leave untouched (reference: rc 123)   */
#define LB2_TREE_DRY_RUN             0x400u /* plan + compact, write nothing                         */
#define LB2_TREE_CLEANUP             0x800u /* also do the script's rm lines (project_build.py:256-259) on the walk */

typedef struct lb2_stats {
  uint32_t n_files, n_ok, n_unsupported, overflow;
  uint64_t in_bytes;          /* input bytes of the n_ok files                                  */
  uint64_t out_bytes;         /* OUT: stripped bytes written                                    */
  uint64_t copy_bytes;        /* C:   extent bytes read (input arena + regenerated literals)    */
  uint64_t header_bytes;      /* H:   header/table/note bytes the planner parsed                */
  uint64_t n_tiles;
  uint64_t out_bytes_needed;  /* 256-byte-rounded arena bytes the batch needs                   */
  float plan_ms;              /* plan + offset scan kernels, CUDA events on the call's stream   */
  float compact_ms;           /* compaction kernel                                              */
  float h2d_ms, d2h_ms;       /* lb2_strip_host only: summed copy time                          */
  uint64_t h2d_bytes;         /* lb2_strip_host only: bytes that crossed the bus upwards (DMA'd ranges, or what the   */
  uint64_t d2h_bytes;         /*   kernels pulled in zero-copy mode) and downwards                                    */
} lb2_stats;

typedef struct lb2_tree_stats {
  uint32_t n_selected;        /* paths whose basename ends in the suffix                        */
  uint32_t n_gpu;             /* replaced with GPU-produced bytes                               */
  uint32_t n_fallback;        /* handed to the host `strip`                                     */
  uint32_t n_skipped;         /* symlinks, directories, tolerated non-ELF                       */
  uint32_t n_failed;          /* would make the reference's script exit non-zero                */
  uint32_t n_removed;         /* LB2_TREE_CLEANUP: *.egg-info, *.dist-info, __pycache__, tests entries removed */
  uint64_t in_bytes, out_bytes;
  double walk_read_s;         /* directory walk + stat                                          */
  double gpu_s;               /* kernels + result fetch, summed over batches                    */
  double write_s;             /* file reads/uploads and downloads/writes (overlapped), wall     */
  double fallback_s;          /* host `strip` on the files the planner refused                  */
  double read_cpu_s;          /* summed over the I/O threads: time inside pread                 */
  double write_cpu_s;         /* ... inside pwrite / truncate                                   */
  double dma_wait_s;          /* ... issuing and waiting for the slot DMAs                      */
  uint32_t io_threads, n_batches;
  lb2_stats batch;
} lb2_tree_stats;

/* ---- context ---------------------------------------------------------------------------- */
int lb2_ctx_create(int device, lb2_ctx **ctx);
void lb2_ctx_destroy(lb2_ctx *ctx);
const char *lb2_last_error(const lb2_ctx *ctx); /* ctx may be NULL: error of the failed create */
const char *lb2_version(void);
int lb2_sm_count(const lb2_ctx *ctx);

/* ---- device / pinned memory for callers without their own CUDA runtime (ctypes) ---------- */
void *lb2_dev_alloc(lb2_ctx *ctx, uint64_t bytes);
void lb2_dev_free(lb2_ctx *ctx, void *p);
void *lb2_pinned_alloc(lb2_ctx *ctx, uint64_t bytes); /* pinned + device-mapped, on the GPU's NUMA node (LB2_NUMA=0: anywhere) */
void lb2_pinned_free(lb2_ctx *ctx, void *p);
int lb2_memcpy_h2d(lb2_ctx *ctx, void *d_dst, const void *h_src, uint64_t bytes);
int lb2_memcpy_d2h(lb2_ctx *ctx, void *h_dst, const void *d_src, uint64_t bytes);
int lb2_memset_d(lb2_ctx *ctx, void *d_dst, int value, uint64_t bytes);
/* device to device; returns when the copy is done, as the two above */
int lb2_memcpy_d2d(lb2_ctx *ctx, void *d_dst, const void *d_src, uint64_t bytes);

/* ---- strip a batch resident in HBM ------------------------------------------------------ */
/* d_in: input arena; file f occupies [h_in_off[f], h_in_off[f+1]) minus padding -- offsets must be
 * multiples of 16 and h_in_sizes[f] gives the exact byte length (NULL: use the offset difference).
 * d_out: output arena of out_capacity bytes; file f lands at out_off[f] (multiples of 256).
 * Enqueues upload of the offsets, the plan kernel, the offset scan and the compaction kernel on
 * `stream` (a cudaStream_t; NULL = the context's own stream) and returns without synchronising.  Up to TWO
 * batches may be in flight (the second is queued behind the first on the stream, so the GPU does not idle while the
 * host collects); lb2_batch_results collects them in order.  Batches that share an output arena overwrite it. */
int lb2_strip_device_async(lb2_ctx *ctx, const void *d_in, const uint64_t *h_in_off, const uint64_t *h_in_sizes,
                           uint32_t n_files, void *d_out, uint64_t out_capacity, uint32_t flags, void *stream);
/* Waits for the OLDEST batch in flight, copies its offsets/status back.  Any pointer may be NULL. */
int lb2_batch_results(lb2_ctx *ctx, uint64_t *h_out_off /* n+1 */, uint64_t *h_out_sizes /* n */,
                      int32_t *h_status /* n */, lb2_stats *stats);

/* ---- strip a shard whose input + output do not fit side by side in HBM ------------------------- */
/* Input arena resident (as above); the output is streamed through a ring of TWO slots of slot_capacity
 * bytes each at d_out_ring: consecutive files are grouped into chunks of <= max_chunk_bytes of arena span
 * (0 = slot_capacity), chunk k is written to slot k % 2 and handed to on_chunk (may be NULL) before the
 * slot is reused two chunks later -- the consumer owns the slot only for the duration of the callback.
 * Offsets passed to the callback are relative to the slot.  h_out_sizes / h_status (n_files each, may be
 * NULL) receive the per-file results; *total sums the chunks (plan_ms / compact_ms: summed kernel times).
 * This is what one `strip` process does to an argument list longer than memory (SURVEY.md D7). */
typedef int (*lb2_chunk_fn)(void *user, uint32_t chunk, uint32_t first_file, uint32_t n_files, const void *d_out_slot,
                            const uint64_t *out_off, const uint64_t *out_sizes, const int32_t *status,
                            const lb2_stats *chunk_stats);
int lb2_strip_device_chunked(lb2_ctx *ctx, const void *d_in, const uint64_t *h_in_off, const uint64_t *h_in_sizes,
                             uint32_t n_files, void *d_out_ring, uint64_t slot_capacity, uint64_t max_chunk_bytes,
                             uint32_t flags, void *stream, lb2_chunk_fn on_chunk, void *user, uint64_t *h_out_sizes,
                             int32_t *h_status, lb2_stats *total);

/* ---- strip a batch held in host memory ---------------------------------------------------- */
/* h_out_off[f] (multiples of 256) and h_out_sizes[f] describe where file f was written in h_out.
 * When both arenas are pinned and device-mapped (lb2_pinned_alloc, cudaHostAlloc, cudaHostRegister) the
 * kernels run on them directly over PCIe (zero-copy: only headers and kept extents are pulled, stripped
 * files are pushed straight back; LB2_HOST_ZEROCOPY=0 disables).  LB2_HOST_DMA=1 selects the copy-engine
 * variant instead: plan over the mapping, DMA of the kept ranges into a device slot, compaction in HBM, DMA
 * of the output (same bytes on the bus).  Otherwise, or when both are
 * disabled: explicit H2D of whole files -> kernels -> D2H, pipelined in <= LB2_CHUNK_MB (256) MB chunks of
 * whole files on three streams.  stats->h2d_bytes / d2h_bytes say what crossed the bus. */
int lb2_strip_host(lb2_ctx *ctx, const void *h_in, const uint64_t *h_in_off, const uint64_t *h_in_sizes,
                   uint32_t n_files, void *h_out, uint64_t out_capacity, uint64_t *h_out_off, uint64_t *h_out_sizes,
                   int32_t *h_status, uint32_t flags, lb2_stats *stats);

/* ---- strip a directory tree in place (the reference's shell line) ------------------------ */
int lb2_strip_tree(lb2_ctx *ctx, const char *root, const char *suffix /* ".so" */, uint32_t flags,
                   lb2_tree_stats *stats);
/* The same with the sibling clean-up lines of the reference's script folded into the directory walk
 * (flag LB2_TREE_CLEANUP; /root/reference/lambdipy/project_build.py:256-259):
 *     rm -rf ROOT/{glob}.egg-info ROOT/{glob}.dist-info          (top level only, shell glob: no dot files)
 *     find ROOT/ -name __pycache__ | xargs rm -rf
 *     find ROOT/ -name tests | grep -v "KEEP" | xargs rm -rf      KEEP = keep_tests_regex, a grep basic regex on
 *                                                                the printed path; the reference passes "*" when
 *                                                                --keep-tests is not given, 'a\|b' otherwise (:249)
 * They run before the selection, as in the script: objects under a removed directory are not stripped. */
int lb2_strip_tree_ex(lb2_ctx *ctx, const char *root, const char *suffix, uint32_t flags, const char *keep_tests_regex,
                      lb2_tree_stats *stats);
/* Only the clean-up lines (no GPU, no context needed). */
int lb2_tree_cleanup(const char *root, const char *keep_tests_regex, uint32_t *n_removed);
/* The `tests` line of the clean-up on paths that are not on disk: removed[i] = 1 when an entry named tests that find
 * prints as lines[i] is removed, 0 when the keep pattern keeps it.  The same rule lb2_tree_cleanup applies. */
int lb2_cleanup_tests_removed(const char *keep_tests_regex, const char *const *lines, uint32_t n, uint8_t *removed);
/* Optional: pay lb2_strip_tree's first-use costs (pinned slot ring, I/O streams, device workspaces) now,
 * e.g. on a helper thread while the reference's script is still running pip
 * (/root/reference/lambdipy/project_build.py:266-268).  expected_tree_bytes sizes the ring (0 = default). */
int lb2_tree_prepare(lb2_ctx *ctx, uint64_t expected_tree_bytes);

/* ---- plan only: per-file output sizes and status, nothing copied (tests) ------------------ */
int lb2_plan_device(lb2_ctx *ctx, const void *d_in, const uint64_t *h_in_off, const uint64_t *h_in_sizes,
                    uint32_t n_files, uint32_t flags, uint64_t *h_out_sizes, int32_t *h_status, lb2_stats *stats);

/* ---- synthetic corpus: fill payload regions of an HBM arena with counter-based random bytes - */
typedef struct lb2_fill_region {
  uint64_t offset; /* byte offset in the arena */
  uint64_t len;
} lb2_fill_region;
/* byte at arena offset o = byte (o & 7) of splitmix64(seed + (o >> 3)); independent of the region
 * split, so host and device generators agree. */
int lb2_corpus_fill(lb2_ctx *ctx, void *d_arena, const lb2_fill_region *h_regions, uint32_t n_regions,
                    uint64_t seed, void *stream);

/* Copies n host-built blobs (ELF headers, notes, string tables) into the arena:
 * arena[h_dst[i] .. +h_len[i]) = h_data[h_src[i] .. +h_len[i]).  Synchronous. */
int lb2_corpus_scatter(lb2_ctx *ctx, void *d_arena, const void *h_data, uint64_t data_bytes, const uint64_t *h_dst,
                       const uint64_t *h_src, const uint64_t *h_len, uint32_t n);

/* ---- gzip writer: raw DEFLATE (RFC 1951) + CRC-32 of a stream fed in pieces ----------------- */
/* What `tarfile.open(path, "w:gz")` spends its time on in PackageBuild.create_compressed_tarball
 * (lambdipy/package_build.py:165-172 of the reference).  The caller writes the gzip header and the
 * CRC32 / ISIZE trailer; the library produces the DEFLATE body between them.
 *
 * Each piece is cut into 64 KB chunks that are deflated independently on the GPU, each looking back
 * 32 KB into the stream (also into earlier pieces), and each ending byte-aligned with an empty stored
 * block (what zlib's Z_SYNC_FLUSH emits).  A chunk is written with dynamic Huffman, fixed Huffman or
 * stored blocks, whichever is smallest, so incompressible data grows by at most LB2_GZIP_BOUND.
 * The same stream always gives the same bytes.
 *
 * Modes (flags of lb2_gzip_create and lb2_zip_create).  0: each chunk is parsed greedily with one-step lazy
 * evaluation over 16 hash-chain candidates per position.  LB2_DEFLATE_BEST: the thorough mode, for archives that are
 * written once and downloaded many times.  After that parse, every chunk is parsed again optimally: each position's
 * Pareto set of matches (up to 8, from up to 1024 hash-chain candidates) and a shortest path over the chunk's
 * positions, priced with the chunk's own Huffman code, four rounds of parse -> code -> prices.  A chunk keeps the
 * smaller of the two parses by the same byte formula, so a best-mode chunk is never larger than the default one; the
 * chunking, flushes, bounds and determinism are those of mode 0.  A best-mode writer holds one workspace of
 * 64 KB x 9 x 4 B = 2.25 MiB per SM of the device (297 MiB on a 132-SM H100) from create to destroy, beside the
 * per-piece buffers both modes hold.
 *
 * Up to TWO pieces may be in flight: lb2_gzip_submit enqueues the upload and the kernels and returns;
 * lb2_gzip_collect waits for the OLDEST piece and copies its compressed bytes out.  h_in must stay
 * unchanged until its piece is collected (pinned memory from lb2_pinned_alloc makes the upload
 * asynchronous).  lb2_gzip_finish appends the final empty block once every piece is collected.
 * Destroy the writer before its context. */
typedef struct lb2_gzip lb2_gzip;
typedef struct lb2_gzip_stats {
  uint64_t in_bytes, out_bytes;      /* stream bytes in; DEFLATE bytes out (final block included)   */
  uint32_t crc32;                    /* CRC-32 of the input collected so far                          */
  uint32_t n_chunks, n_stored_chunks, n_fixed_chunks;  /* 64 KB chunks; those written stored / fixed Huffman */
  float deflate_ms;                  /* deflate + compaction kernels, CUDA events, summed over pieces */
  float crc_ms;                      /* CRC-32 kernel                                                 */
  float h2d_ms;                      /* piece uploads, or the gathers of device pieces (CUDA events)  */
  float d2h_ms;                      /* result downloads (host clock around the copy)                 */
  uint32_t n_opt_chunks;             /* chunks written from the optimal parse (0 in the default mode) */
  float best_ms;                     /* best mode: the optimal-parse kernel (also in deflate_ms)      */
} lb2_gzip_stats;
#define LB2_DEFLATE_BEST 1u          /* lb2_gzip_create / lb2_zip_create: the thorough mode (above)   */
/* worst-case DEFLATE bytes of one piece of n input bytes (out_cap of lb2_gzip_collect) */
#define LB2_GZIP_BOUND(n) ((n) + 15 * (((n) + 65535) / 65536))
int lb2_gzip_create(lb2_ctx *ctx, uint32_t flags /* 0 or LB2_DEFLATE_BEST */, lb2_gzip **g);
int lb2_gzip_submit(lb2_gzip *g, const void *h_in, uint64_t n);
/* LB2_E_CAPACITY when out_cap is too small: *out_n says how much is needed, the piece stays in flight */
int lb2_gzip_collect(lb2_gzip *g, void *h_out, uint64_t out_cap, uint64_t *out_n);
/* writes the final block (2 bytes); *crc32 / *isize (full length; gzip stores it mod 2^32) for the trailer */
int lb2_gzip_finish(lb2_gzip *g, void *h_out, uint64_t out_cap, uint64_t *out_n, uint32_t *crc32, uint64_t *isize,
                    lb2_gzip_stats *stats);
/* A piece whose bytes are already in device memory, which is how tarball.strip_tarball strips the shared objects inside
 * a .tar.gz without the tar stream leaving the device.  The piece is src[0].len + ... + src[n_segs - 1].len bytes: the
 * segments (lb2_zip_source, of any alignment) back to back, with no padding.  A gather kernel on the writer's stream
 * lays them out in the piece buffer; from there the piece is what lb2_gzip_submit makes of the concatenation -- the
 * same chunks, history, CRC-32, ISIZE, bytes out and LB2_E_STATE cases (stats.h2d_ms then times the gather).
 * n_segs may be 0 (an empty piece).  The caller guarantees that the sources are complete when this is called and
 * leaves them unchanged until the piece is collected. */
struct lb2_zip_source;
int lb2_gzip_submit_device(lb2_gzip *g, const struct lb2_zip_source *src, uint32_t n_segs);
/* The compressed size of every 64 KB chunk of the piece collected last, in stream order: sizes[0 .. *n_chunks), which
 * sum to that collect's *out_n (an empty piece has none).  Chunk i of a piece of n bytes holds its bytes
 * [64 KB * i, min(n, 64 KB * (i + 1))), and every chunk ends byte-aligned with an empty stored block, so the next
 * one starts a block at a known byte: what a seek table records (seek_table.py).  Call it after lb2_gzip_collect and
 * before the next submit reuses that piece's slot (LB2_E_STATE otherwise); LB2_E_CAPACITY when cap is too small
 * (*n_chunks says how many).  The final block that lb2_gzip_finish writes is not part of any chunk. */
int lb2_gzip_chunk_sizes(lb2_gzip *g, uint32_t *sizes, uint32_t cap, uint32_t *n_chunks);
void lb2_gzip_destroy(lb2_gzip *g);

/* ---- zip writer: one raw DEFLATE stream + CRC-32 per file, many files per piece ------------------ */
/* What `shutil.make_archive(base, "zip", "./build")` spends its time on when a Lambda bundle is zipped: every
 * zip member is its own raw DEFLATE stream.  The caller writes the zip container (headers, central directory);
 * the library produces each member's body and CRC-32.
 *
 * A piece holds n_segs segments, one per file (or part of a file): segment i is h_in[seg_off[i] ..
 * + seg_len[i]), seg_off[i] a multiple of 16, in increasing order without overlap.  Each segment is deflated
 * like a gzip piece (64 KB chunks, sync-flushed, dynamic / fixed / stored per chunk), but no chunk crosses a
 * segment and no match reaches into another file; a file that ends in the piece is closed with the 2-byte final
 * block 03 00, so an empty file's body is exactly 03 00 (as zlib's); flags select the mode, as for lb2_gzip_create.
 * Each member costs at most 5 + 2 bytes of
 * framing per 64 KB chunk, plus 2 for its final block, over its stored size.
 *
 * A file larger than a piece continues into the next one: submit its first part as the LAST segment with
 * LB2_ZIP_MORE, and its rest as segment 0 (seg_off[0] = 0) of the next piece with LB2_ZIP_CONTINUES; the
 * library keeps the file's last 32 KB on the device as history and its running CRC-32.  Chunks start at
 * multiples of 64 KB of each segment, so cut a file at a multiple of 64 KB of its bytes: it is then deflated in
 * the chunks (and within the bound) of the whole file; a cut elsewhere costs one more chunk per piece boundary.
 *
 * Up to TWO pieces may be in flight, as with lb2_gzip_*.  lb2_zip_collect waits for the OLDEST piece, copies
 * its DEFLATE bytes (all segments back to back) to h_out and fills segs[0 .. n_segs) of that piece: where each
 * segment's bytes are in h_out, the CRC-32 of its file from the file's first byte (earlier pieces included),
 * and whether the file ended.  stats (may be NULL) receives the totals so far; its crc32 is the running CRC-32
 * of the file left open (0 if none).  The same pieces always give the same bytes.  Destroy the writer before its
 * context. */
typedef struct lb2_zip lb2_zip;
typedef struct lb2_zip_segment {
  uint64_t out_off, out_len;   /* the segment's DEFLATE bytes in the collected output                       */
  uint32_t crc32;              /* CRC-32 of the file so far                                                 */
  uint32_t ended;              /* 1: the file ended in this piece; its bytes end with the final block       */
} lb2_zip_segment;
#define LB2_ZIP_CONTINUES 1u   /* segment 0 continues the file the previous piece left open                 */
#define LB2_ZIP_MORE      2u   /* the last segment's file continues in the next piece                       */
/* worst-case DEFLATE bytes of one piece of n bytes (padding included) in n_segs segments (out_cap of lb2_zip_collect) */
#define LB2_ZIP_BOUND(n, n_segs) (LB2_GZIP_BOUND(n) + 17 * (uint64_t)(n_segs))
int lb2_zip_create(lb2_ctx *ctx, uint32_t flags /* 0 or LB2_DEFLATE_BEST */, lb2_zip **z);
/* LB2_E_STATE: two pieces in flight, LB2_ZIP_CONTINUES without an open file, or an open file not continued */
int lb2_zip_submit(lb2_zip *z, const void *h_in, uint64_t n, const uint64_t *seg_off, const uint64_t *seg_len,
                   uint32_t n_segs, uint32_t flags);
/* LB2_E_CAPACITY when out_cap is too small: *out_n says how much is needed, the piece stays in flight */
int lb2_zip_collect(lb2_zip *z, void *h_out, uint64_t out_cap, uint64_t *out_n, lb2_zip_segment *segs,
                    lb2_gzip_stats *stats);
/* A piece whose segments are already in device memory -- the output of lb2_unzip_run or of a strip call, which is how
 * zipfile_gpu.strip_zip strips the shared objects inside a zip (what `extractall`, the reference's
 * `find -name "*.so" | xargs strip` and `make_archive` do in three passes over the file system) without the decoded
 * bytes leaving the device.  Segment i is src[i].len bytes at src[i].d_ptr, of any alignment.  A gather kernel on the
 * writer's stream lays the segments out at 16-byte-aligned offsets of the piece, in order, and zeroes the gaps; from
 * there the piece is what lb2_zip_submit makes of the same segments -- the same chunks, history, flags, states and
 * LB2_E_STATE cases, collected by lb2_zip_collect, with the same bytes out (stats.h2d_ms then times the gather).
 * The caller guarantees that the sources are complete when this is called (lb2_unzip_run and lb2_batch_results both
 * end in a host wait) and leaves them unchanged until the piece is collected. */
typedef struct lb2_zip_source {
  const void *d_ptr;           /* device memory                                                             */
  uint64_t len;                /* bytes; 0 for an empty file (d_ptr may then be NULL)                       */
} lb2_zip_source;
int lb2_zip_submit_device(lb2_zip *z, const lb2_zip_source *src, uint32_t n_segs, uint32_t flags);
/* lb2_gzip_chunk_sizes for the zip writer: the compressed size of every 64 KB chunk of the piece collected last, in
 * segment order (a segment of n bytes has max(1, ceil(n / 64 KB)) chunks, cut at multiples of 64 KB of the segment;
 * the last chunk of a file that ended includes its final block 03 00).  Each segment's sizes sum to its out_len. */
int lb2_zip_chunk_sizes(lb2_zip *z, uint32_t *sizes, uint32_t cap, uint32_t *n_chunks);
void lb2_zip_destroy(lb2_zip *z);

/* ---- gzip reader: raw DEFLATE (RFC 1951) decoded on the GPU ----------------------------------- */
/* What `tarfile.open(path, "r:gz")` spends its time on in prepare_tarfile (lambdipy/project_build.py:98-102 of the
 * reference).  The caller parses the gzip header and trailer; the library decodes the DEFLATE body in between.
 *
 * Any valid stream decodes, also one with no flush points: the body is cut into spans of LB2_INFLATE_SPAN_KB (read
 * at each call, default 128) compressed KB; each span after the first starts at a block-header candidate found by
 * search, is decoded speculatively, and is used only if its start is where the span before it ended (otherwise it
 * is decoded again from that confirmed position).  Invalid or truncated input gives LB2_E_DATA, never other bytes.
 * Device memory: the body plus about 3 bytes per decoded byte (LB2_E_CAPACITY when that does not fit).
 *
 * lb2_inflate_run decodes the stream that starts at h_in; bytes after its final block (a gzip trailer, further
 * members) are ignored, and stats.in_bytes says where the stream ended.  The decoded bytes stay on the device until
 * lb2_inflate_read copies them out (the next run replaces them).  Destroy the reader before its context. */
typedef struct lb2_inflate lb2_inflate;
typedef struct lb2_inflate_stats {
  uint64_t in_bytes, out_bytes;   /* DEFLATE bytes consumed (to the end of the final block), bytes produced       */
  uint32_t crc32;                 /* CRC-32 of the decoded bytes                                                  */
  uint32_t n_spans;               /* spans decoded on their own                                                   */
  uint32_t n_rounds;              /* count rounds of the chain                                                    */
  uint32_t n_rejected;            /* candidates the chain rejected (a wrong start, decoded again from the right one) */
  uint32_t n_absorbed;            /* nominal spans without a candidate, decoded by the span before them          */
  float find_ms, count_ms, decode_ms, resolve_ms, crc_ms;  /* kernel times (CUDA events), count summed over rounds */
  float h2d_ms;                   /* body upload (CUDA events)                                                    */
} lb2_inflate_stats;
int lb2_inflate_create(lb2_ctx *ctx, uint32_t flags /* 0 */, lb2_inflate **d);
/* decode the raw DEFLATE stream at h_in (at most n bytes) on the device; *out_n = its exact decoded size */
int lb2_inflate_run(lb2_inflate *d, const void *h_in, uint64_t n, uint64_t *out_n, lb2_inflate_stats *stats);
/* copy the decoded bytes of the last successful run to h_out (cap >= *out_n) */
int lb2_inflate_read(lb2_inflate *d, void *h_out, uint64_t cap);
/* The device buffer lb2_inflate_read would copy from: *n bytes at *d_out (NULL when *n is 0), 256-byte aligned.  Valid
 * until the next lb2_inflate_run or lb2_inflate_destroy.  LB2_E_STATE without a successful run. */
int lb2_inflate_device_output(lb2_inflate *d, const void **d_out, uint64_t *n);
/* A stream with a seek table (seek_table.py): spans[i] is the compressed and the decoded length of a run of the
 * stream, in order from its first byte; every run after the first starts with a block header at its first byte.  Each
 * run is decoded once, by one thread, from its known start into its known output range (lb2_inflate_table_decode_
 * kernel): no candidate search, no count rounds.  The table is outside input.  It is refused without a launch when an
 * entry is 0, decodes to more than 1032 bytes per compressed byte or the runs pass n; it is refused after the decode
 * unless every run decoded exactly its length and ended at the block header the next run starts at, and only the last
 * run decoded the final block, ending with the table's last byte.  An accepted table therefore gives exactly the
 * stream's DEFLATE decode; a refused one is followed by the search of lb2_inflate_run on the same stream.  Either way
 * the bytes, CRC-32, return code and stats.in_bytes are what lb2_inflate_run gives: a lying table costs time, never a
 * different result.  *n_table = 1 when the stream was decoded from the table (stats: 0 find and count rounds,
 * n_spans = the entries), *n_refused = 1 when a table was given and refused (both may be NULL). */
typedef struct lb2_inflate_span {
  uint64_t in_len, out_len;       /* compressed bytes, decoded bytes                                              */
} lb2_inflate_span;
int lb2_inflate_run_table(lb2_inflate *d, const void *h_in, uint64_t n, const lb2_inflate_span *spans, uint32_t n_spans,
                          uint64_t *out_n, lb2_inflate_stats *stats, uint32_t *n_table, uint32_t *n_refused);
void lb2_inflate_destroy(lb2_inflate *d);

/* ---- zip reader: every member of a zip decoded and checked on the GPU in one batch ------------------ */
/* What `ZipFile.extractall` and `ZipFile.testzip` spend their time on.  The caller parses the zip (central directory
 * and local headers) and uploads a buffer holding the member bodies; the library decodes every member and computes
 * its CRC-32 on the device.  Each member is its own raw DEFLATE stream (method 8) or stored as it is (method 0).
 *
 * members[i] names the body h_in[body_off .. body_off + body_len) and the size and CRC-32 the archive records for
 * it.  Member i's output is placed at results[i].out_off: the exclusive scan of the sizes, each rounded up to 16
 * bytes.  Every bit a decoder reads is bounded by the member's own body.  A DEFLATE body of at most one span
 * (LB2_INFLATE_SPAN_KB, read at each call, default 128) is decoded whole by one thread straight into its output; a
 * larger one runs the speculative span pipeline of lb2_inflate_run, its spans batched with every other member's in
 * each launch.  STORED bodies are copied on the device.
 *
 * results[i].status is the member's own: LB2_UNZIP_OK, LB2_UNZIP_BAD_DATA (invalid or truncated DEFLATE),
 * LB2_UNZIP_WRONG_SIZE (more or fewer bytes than out size; a STORED body whose length is not its size) or
 * LB2_UNZIP_BAD_CRC (results[i].crc32, computed on the device, differs from the member's crc32).  A bad member never
 * changes another member's bytes or status, and the run itself still returns LB2_OK.
 *
 * Everything in the table is checked before any launch: a method other than 0 or 8, a body outside [0, n) or output
 * sizes that overflow give LB2_E_ARG; a batch that does not fit in device memory (about n + 3 bytes per output byte
 * when a member takes the span pipeline, n + 1 otherwise) gives LB2_E_CAPACITY.  The decoded bytes stay on the device
 * until lb2_unzip_read copies them out (the next run replaces them).  Destroy the reader before its context. */
typedef struct lb2_unzip lb2_unzip;
typedef struct lb2_unzip_member {
  uint64_t body_off, body_len;    /* the member's body in h_in                                                   */
  uint64_t size;                  /* uncompressed size, from the central directory                               */
  uint32_t crc32;                 /* CRC-32, from the central directory                                          */
  uint32_t method;                /* 0 (stored) or 8 (DEFLATE)                                                   */
} lb2_unzip_member;
#define LB2_UNZIP_OK 0
#define LB2_UNZIP_BAD_DATA 1
#define LB2_UNZIP_WRONG_SIZE 2
#define LB2_UNZIP_BAD_CRC 3
typedef struct lb2_unzip_result {
  uint64_t out_off;               /* the member's bytes in the lb2_unzip_read buffer                             */
  uint32_t crc32;                 /* CRC-32 of those bytes (meaningful when the status is OK or BAD_CRC)         */
  int32_t status;                 /* LB2_UNZIP_*                                                                 */
} lb2_unzip_result;
typedef struct lb2_unzip_stats {
  uint64_t in_bytes, out_bytes;   /* buffer bytes uploaded, sum of the member sizes                              */
  uint32_t n_members, n_stored, n_small, n_large;  /* members in all and on each path (copy, one span, pipeline) */
  uint32_t n_spans;               /* spans the larger members were decoded in                                    */
  uint32_t n_rounds;              /* count rounds (every chain advances in each)                                 */
  uint32_t n_rejected, n_absorbed; /* as in lb2_inflate_stats, summed over the members                           */
  uint32_t n_bad;                 /* members whose status is not LB2_UNZIP_OK                                    */
  float h2d_ms, copy_ms, small_ms, find_ms, count_ms, decode_ms, resolve_ms, crc_ms;  /* CUDA events             */
} lb2_unzip_stats;
int lb2_unzip_create(lb2_ctx *ctx, uint32_t flags /* 0 */, lb2_unzip **u);
/* decode members[0 .. n_members) of the buffer h_in (n bytes); *out_n = bytes lb2_unzip_read copies out */
int lb2_unzip_run(lb2_unzip *u, const void *h_in, uint64_t n, const lb2_unzip_member *members, uint32_t n_members,
                  uint64_t *out_n, lb2_unzip_result *results, lb2_unzip_stats *stats);
/* copy the output of the last successful run to h_out (cap >= *out_n) */
int lb2_unzip_read(lb2_unzip *u, void *h_out, uint64_t cap);
/* The device buffer lb2_unzip_read would copy from, *n bytes at *d_out (NULL when *n is 0): member i's bytes are at
 * results[i].out_off, a multiple of 16, which is what lb2_strip_device_async wants of an input arena and what
 * lb2_zip_submit_device takes as a source.  Valid until the next lb2_unzip_run or lb2_unzip_destroy.  LB2_E_STATE
 * without a successful run. */
int lb2_unzip_device_output(lb2_unzip *u, const void **d_out, uint64_t *n);
/* lb2_unzip_run with seek tables (seek_table.py): member i's entries are spans[span_first[i] .. span_first[i + 1])
 * (none: no table; span_first has n_members + 1 entries).  A DEFLATE member larger than one span whose entries add up
 * to its body and size is decoded from its table as in lb2_inflate_run_table, in one launch with every other table
 * member's spans; members without a table, with a table that is refused before or after the decode, and one-span
 * members (decoded whole by one thread, no search to save) take the path they take in lb2_unzip_run, in the same
 * batch and into the same output.  Results, statuses and CRC-32s are lb2_unzip_run's; *n_table / *n_refused (may be
 * NULL) count the members decoded from a table and the tables refused. */
int lb2_unzip_run_table(lb2_unzip *u, const void *h_in, uint64_t n, const lb2_unzip_member *members, uint32_t n_members,
                        const uint32_t *span_first, const lb2_inflate_span *spans, uint64_t *out_n,
                        lb2_unzip_result *results, lb2_unzip_stats *stats, uint32_t *n_table, uint32_t *n_refused);
void lb2_unzip_destroy(lb2_unzip *u);

/* ---- tar index: the bytes tarfile reads to list the members of a tar stream in device memory ---------------- */
/* One warp walks the headers of d_tar[0 .. n) (16-byte aligned) the way Python 3.12's tarfile lists members (USTAR,
 * GNU, PAX and v7 headers; GNU long names, pax records of up to 1 MiB, GNU old-sparse extension blocks) and gathers
 * every range that listing reads: each header block, the byte in front of it (TarFile.next reads it to check that the
 * previous member's data exists), the extended headers' data, and the block where the walk stopped (an all-zero
 * block, a header tarfile refuses, the end of the data, or something the walk does not follow).  ranges[0 .. *n_ranges)
 * are sorted, do not touch each other, and their bytes are in h_bytes[0 .. *n_bytes) back to back.  A caller that
 * lists the members with tarfile from these bytes reads nothing else on the archives people have, and fetches
 * whatever else it reads.
 * LB2_E_CAPACITY when max_ranges or bytes_cap is too small: *n_ranges / *n_bytes say what is needed, stats is filled. */
typedef struct lb2_tar_range {
  uint64_t off, len;
} lb2_tar_range;
#define LB2_TAR_STOP_ZERO 1          /* an all-zero block: the end-of-archive marker                                  */
#define LB2_TAR_STOP_BAD_HEADER 2    /* a bad checksum or a number field tarfile refuses                              */
#define LB2_TAR_STOP_END 3           /* the end of the data, inside or right at a header                              */
#define LB2_TAR_STOP_UNSUPPORTED 4   /* an extended header over 1 MiB, pax records the walk does not follow          */
typedef struct lb2_tar_index_stats {
  uint64_t n_members;      /* member headers walked (extended headers not counted)                                  */
  uint64_t stop_offset;    /* the offset of the block the walk stopped at                                           */
  uint32_t stop_reason;    /* LB2_TAR_STOP_*                                                                        */
  float kernel_ms;         /* the walk kernel (CUDA events)                                                         */
} lb2_tar_index_stats;
int lb2_tar_index(lb2_ctx *ctx, const void *d_tar, uint64_t n, lb2_tar_range *ranges, uint32_t max_ranges,
                  uint32_t *n_ranges, void *h_bytes, uint64_t bytes_cap, uint64_t *n_bytes, lb2_tar_index_stats *stats);

/* ---- dynamic sections: what the loader reads of shared objects in device memory ------------------------------ */
/* What `readelf -dW` and `readelf -VW` print of each shared object's dependencies -- DT_SONAME, DT_NEEDED, DT_RPATH,
 * DT_RUNPATH, the version needs and the version definitions -- read where the objects lie, which is how
 * deps.check_zip tells whether the shared objects of a Lambda zip will load (where the host would inflate every
 * object, or bring it back over PCIe, and run readelf on it).  Object i is sizes[i] bytes at the device address
 * d_ptrs[i] (both arrays in host memory; any alignment), such as the (address, size) pairs lb2_unzip_device_output
 * hands out.  One warp parses each object (kernels in elf_deps.cu, logic in elf_deps.cuh): the ELF header, the
 * program headers, the dynamic array up to DT_NULL or PT_DYNAMIC's end, and the DT_VERNEED / DT_VERDEF chains, with
 * addresses mapped through the PT_LOADs.  No byte outside an object's [0, size) is read.
 *
 * objects[i] receives the status, e_machine / e_type and where its records and strings are: records[first_record ..
 * first_record + n_records), in this order -- the string tags in dynamic-array order (DT_NEEDED in the loader's
 * order), then each Verneed as a VERNEED_FILE record followed by its VERNEED_VERSION records, then the first name of
 * each Verdef as a VERDEF record -- and their strings, each followed by a NUL, in h_pool[pool_off .. pool_off +
 * pool_len).  Only LB2_ELF_OK objects have records.  LB2_E_CAPACITY when max_records or pool_cap is too small:
 * objects[] and stats are filled and *n_records / *pool_bytes say what is needed.  stats.kernel_ms times the two
 * passes (count, then write at the host's exclusive scan of the counts) with CUDA events. */
#define LB2_ELF_OK 0
#define LB2_ELF_NOT_ELF 1            /* no ELF magic                                                                  */
#define LB2_ELF_UNSUPPORTED 2        /* ELF32 or big-endian: not parsed                                               */
#define LB2_ELF_STATIC 3             /* no PT_DYNAMIC                                                                 */
#define LB2_ELF_MALFORMED 4          /* an offset, address or link outside the file or its segment, a string not     */
                                     /* ended before DT_STRSZ, a chain cut short of its count or past n / 8 entries  */
#define LB2_ELF_REC_SONAME 1
#define LB2_ELF_REC_NEEDED 2
#define LB2_ELF_REC_RPATH 3
#define LB2_ELF_REC_RUNPATH 4
#define LB2_ELF_REC_VERNEED_FILE 5     /* vn_file                                                                      */
#define LB2_ELF_REC_VERNEED_VERSION 6  /* vna_name; flags = vna_flags (2: weak), ref = its VERNEED_FILE record       */
#define LB2_ELF_REC_VERDEF 7           /* the first vda_name of a Verdef; flags = vd_flags (1: the base version)      */
typedef struct lb2_elf_object {
  int32_t status;                 /* LB2_ELF_*                                                                    */
  uint16_t machine, type;         /* e_machine, e_type (0 unless the header is a complete ELF64 little-endian one) */
  uint32_t first_record, n_records;
  uint64_t pool_off, pool_len;
} lb2_elf_object;
typedef struct lb2_elf_record {
  uint32_t kind;                  /* LB2_ELF_REC_*                                                                */
  uint32_t flags, ref;
  uint32_t len;                   /* the string's bytes, without its NUL                                          */
  uint64_t off;                   /* the string in h_pool                                                         */
} lb2_elf_record;
typedef struct lb2_elf_deps_stats {
  uint64_t n_records, pool_bytes; /* needed, also past the capacities                                             */
  uint64_t bytes_down;            /* device-to-host bytes: the objects, records and pool                          */
  float kernel_ms;                /* the count and write kernels (CUDA events)                                    */
} lb2_elf_deps_stats;
int lb2_elf_deps(lb2_ctx *ctx, const uint64_t *d_ptrs, const uint64_t *sizes, uint32_t n, lb2_elf_object *objects,
                 lb2_elf_record *records, uint32_t max_records, uint32_t *n_records, void *h_pool, uint64_t pool_cap,
                 uint64_t *pool_bytes, lb2_elf_deps_stats *stats);

/* ---- symbol lookups: the undefined symbols a shared object binds when it is loaded ---------------------------- */
/* What ld.so's relocation of an object looks up (glibc elf/dl-lookup.c do_lookup_x and check_match), done for many
 * objects at once, which is how deps.check_zip(symbols=True) finds the "undefined symbol" a dlopen would fail on.
 * A resolver (lb2_syms) owns a device arena that outlives the objects it indexed.
 *
 * lb2_syms_index: objects i < n lie at the device addresses d_ptrs[i] (sizes[i] bytes; both arrays in host memory;
 * any alignment).  One warp per object reads its dynamic array, copies .dynsym, .dynstr, .gnu.version, its hash table
 * (DT_GNU_HASH, else DT_HASH) and its version table into the arena, and lists its references: the symbols that a
 * DT_RELA or DT_JMPREL entry names which are SHN_UNDEF and not STB_LOCAL.  ids[i] receives the object's id in the
 * resolver, objects[i] its status (LB2_SYM_*) and counts.  No byte outside an object's [0, size) is read, and the
 * object may be freed when the call returns.  LB2_E_CAPACITY when the arena cannot grow (nothing was added).
 *
 * lb2_syms_resolve: job j looks up every reference of object jobs[j].obj in the scope scope[scope_off ..+ scope_len)
 * (object ids, in lookup order), one warp per (reference, job).  counts[3 j + classes[id]] counts the references the
 * object `id` defined first in scope order (classes: one byte per id, 0 .. 2).  A strong reference defined nowhere is
 * a miss {job, ref}, in no particular order; *n_misses says how many there were, LB2_E_CAPACITY when more than
 * max_misses (counts are then complete).  Weak references found nowhere are counted nowhere.
 *
 * lb2_syms_names: the strings of misses[0 .. n): for miss i, h_pool[offsets[i] ..] holds its symbol name, the name of
 * the version it asks for and the file of that version need, each followed by a NUL (empty when not versioned).
 * LB2_E_CAPACITY when pool_cap is too small (*pool_bytes says what is needed).
 *
 * lb2_syms_find: what dlsym(handle, name) returns, for names the host gives (deps.check_zip(python=...) looks up each
 * extension module's PyInit_* this way).  Query q looks the name h_names[name_off ..+ name_len) up in the scope
 * scope[scope_off ..+ scope_len) (object ids: the handle's local scope, the object and its DT_NEEDED closure breadth
 * first), one warp per query, with the rules of lb2_syms_resolve for an unversioned lookup under
 * DL_LOOKUP_RETURN_NEWEST: a definition at versym index 0 or 1 is taken, one at index 2 or above only when it is not
 * hidden and the object's single such candidate.  found[q] is the first object in scope order that defines it: its id,
 * the symbol's index, st_info, st_other and versym (0 without DT_VERSYM); obj is LB2_SYM_NOT_FOUND when none does.
 * Only the names go up and only found[] comes down; stats.resolve_ms times the kernel.  LB2_E_ARG for a query outside
 * the name pool or the scope array, or a scope entry that is not an object id. */
#define LB2_SYM_OK 0
#define LB2_SYM_NOT_ELF 1
#define LB2_SYM_UNSUPPORTED 2        /* ELF32, big-endian, or DT_REL relocations                                     */
#define LB2_SYM_STATIC 3
#define LB2_SYM_MALFORMED 4          /* elf_deps' bounds rules, a hash table or a relocation symbol index outside its */
                                     /* table, DT_SYMENT != 24, DT_RELAENT != 24, a reference name not ended          */
typedef struct lb2_syms lb2_syms;
typedef struct lb2_sym_object {
  int32_t status;                    /* LB2_SYM_*                                                                  */
  uint32_t flags;                    /* 1: DT_GNU_HASH, 2: DT_HASH, 4: DT_VERSYM                                   */
  uint32_t nsyms, nver;              /* symbols copied (the hash table's, or past it up to the top relocation's)   */
  uint32_t nbucket, symoffset, bloom_words, bloom_shift;
  uint32_t nrefs, nhash;             /* references; symbols the hash table covers                                   */
  uint64_t str_len, hash_len;
  uint64_t sym_off, str_off, versym_off, hash_off;
  uint64_t rela_off, rela_n, plt_off, plt_n;
  uint64_t arena, refs;              /* device addresses of its tables and references                              */
} lb2_sym_object;
typedef struct lb2_sym_job {
  uint32_t obj, scope_off, scope_len, pad;
} lb2_sym_job;
typedef struct lb2_sym_miss {
  uint32_t job, ref;
} lb2_sym_miss;
#define LB2_SYM_NOT_FOUND 0xffffffffu
typedef struct lb2_sym_query {
  uint32_t scope_off, scope_len;     /* the scope: scope[scope_off ..+ scope_len)                                  */
  uint32_t name_off, name_len;       /* the name: h_names[name_off ..+ name_len), no NUL needed                     */
} lb2_sym_query;
typedef struct lb2_sym_found {
  uint32_t obj, sym;                 /* the defining object's id (LB2_SYM_NOT_FOUND: none) and the symbol's index   */
  uint8_t info, other;               /* its st_info, st_other                                                       */
  uint16_t versym;                   /* its .gnu.version entry, 0 without DT_VERSYM                                 */
} lb2_sym_found;
typedef struct lb2_syms_stats {
  uint64_t bytes_up, bytes_down;     /* host-device bytes of the call                                              */
  uint64_t references, lookups;      /* references indexed or resolved; scope entries probed                        */
  uint64_t arena_bytes;              /* the arena's size after the call                                            */
  float index_ms, refs_ms, resolve_ms; /* kernels (CUDA events)                                                    */
  float pad;
} lb2_syms_stats;
int lb2_syms_create(lb2_ctx *ctx, lb2_syms **out);
void lb2_syms_destroy(lb2_syms *s);
int lb2_syms_index(lb2_syms *s, const uint64_t *d_ptrs, const uint64_t *sizes, uint32_t n, uint32_t *ids,
                   lb2_sym_object *objects, lb2_syms_stats *stats);
int lb2_syms_resolve(lb2_syms *s, const lb2_sym_job *jobs, uint32_t n_jobs, const uint32_t *scope, uint32_t n_scope,
                     const uint8_t *classes, uint32_t *counts, lb2_sym_miss *misses, uint32_t max_misses,
                     uint32_t *n_misses, lb2_syms_stats *stats);
int lb2_syms_names(lb2_syms *s, const lb2_sym_job *jobs, uint32_t n_jobs, const lb2_sym_miss *misses, uint32_t n,
                   uint64_t *offsets, void *h_pool, uint64_t pool_cap, uint64_t *pool_bytes, lb2_syms_stats *stats);
int lb2_syms_find(lb2_syms *s, const lb2_sym_query *queries, uint32_t n, const uint32_t *scope, uint32_t n_scope,
                  const void *h_names, uint64_t names_bytes, lb2_sym_found *found, lb2_syms_stats *stats);

#ifdef __cplusplus
}
#endif
#endif
