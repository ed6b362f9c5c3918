"""ctypes binding of liblambdipy_b200.so (C ABI: include/lambdipy_b200.h).

The library is CUDA-only: there is no CPU implementation behind it, and nothing here falls back
to one.  `load()` raises if the shared object is missing (build it with
`python -m lambdipy_b200.build`); `Context()` raises `NoDeviceError` without an H100.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LAMBDIPY_B200_LIB") or os.path.join(_HERE, "liblambdipy_b200.so")  # (override: diagnostic builds)

# return codes / status / flags (mirror include/lambdipy_b200.h)
LB2_OK, LB2_E_CUDA, LB2_E_ARG, LB2_E_CAPACITY, LB2_E_IO, LB2_E_NODEVICE, LB2_E_STATE, LB2_E_DATA = 0, -1, -2, -3, -4, -5, -6, -7
ST_OK, ST_NOT_ELF, ST_NOT_ELF64LE, ST_BAD_TYPE, ST_NO_SECTIONS, ST_XINDEX = 0, 1, 2, 3, 4, 5
ST_UNSUPPORTED_LAYOUT, ST_BAD_NOTES, ST_PLANNER_LIMIT, ST_MALFORMED = 6, 7, 8, -1
F_NO_MERGE_NOTES = 1
TREE_FALLBACK_HOST_STRIP, TREE_TOLERATE_NON_ELF, TREE_DRY_RUN, TREE_CLEANUP = 0x100, 0x200, 0x400, 0x800

EXPORTS = [
    "lb2_ctx_create", "lb2_ctx_destroy", "lb2_last_error", "lb2_version", "lb2_sm_count",
    "lb2_dev_alloc", "lb2_dev_free", "lb2_pinned_alloc", "lb2_pinned_free",
    "lb2_memcpy_h2d", "lb2_memcpy_d2h", "lb2_memset_d",
    "lb2_strip_device_async", "lb2_batch_results", "lb2_strip_host", "lb2_strip_tree",
    "lb2_plan_device", "lb2_corpus_fill", "lb2_corpus_scatter",
    "lb2_strip_device_chunked", "lb2_tree_prepare", "lb2_strip_tree_ex", "lb2_tree_cleanup",
    "lb2_gzip_create", "lb2_gzip_submit", "lb2_gzip_collect", "lb2_gzip_finish", "lb2_gzip_destroy",
    "lb2_inflate_create", "lb2_inflate_run", "lb2_inflate_read", "lb2_inflate_destroy",
    "lb2_zip_create", "lb2_zip_submit", "lb2_zip_collect", "lb2_zip_destroy",
    "lb2_unzip_create", "lb2_unzip_run", "lb2_unzip_read", "lb2_unzip_destroy",
    "lb2_zip_submit_device", "lb2_unzip_device_output",
    "lb2_inflate_device_output", "lb2_memcpy_d2d", "lb2_gzip_submit_device", "lb2_tar_index",
    "lb2_gzip_chunk_sizes", "lb2_inflate_run_table", "lb2_zip_chunk_sizes", "lb2_unzip_run_table",
    "lb2_cleanup_tests_removed", "lb2_elf_deps",
    "lb2_syms_create", "lb2_syms_destroy", "lb2_syms_index", "lb2_syms_resolve", "lb2_syms_names", "lb2_syms_find",
]
TAR_STOP_ZERO, TAR_STOP_BAD_HEADER, TAR_STOP_END, TAR_STOP_UNSUPPORTED = 1, 2, 3, 4
ZIP_CONTINUES, ZIP_MORE = 1, 2
ELF_OK, ELF_NOT_ELF, ELF_UNSUPPORTED, ELF_STATIC, ELF_MALFORMED = 0, 1, 2, 3, 4  # LB2_ELF_*
ELF_REC_SONAME, ELF_REC_NEEDED, ELF_REC_RPATH, ELF_REC_RUNPATH = 1, 2, 3, 4  # LB2_ELF_REC_*
ELF_REC_VERNEED_FILE, ELF_REC_VERNEED_VERSION, ELF_REC_VERDEF = 5, 6, 7
SYM_OK, SYM_UNSUPPORTED, SYM_MALFORMED = 0, 2, 4  # LB2_SYM_* (the LB2_ELF_* values)
SYM_NOT_FOUND = 0xFFFFFFFF  # LB2_SYM_NOT_FOUND
DEFLATE_BEST = 1  # LB2_DEFLATE_BEST


def deflate_flags(compresslevel):
    """The lb2_gzip_create / lb2_zip_create flags of a writer's `compresslevel`: None keeps the default encoder, 9
    selects the thorough mode (LB2_DEFLATE_BEST, an optimal parse).  There are no levels 1-8."""
    if compresslevel is None:
        return 0
    if type(compresslevel) is int and compresslevel == 9:
        return DEFLATE_BEST
    raise ValueError("compresslevel=%r: expected None (the default encoder) or 9 (the optimal parse)" % (compresslevel,))


def gzip_bound(n):
    """worst-case DEFLATE bytes of one gzip piece of n input bytes (LB2_GZIP_BOUND)"""
    return n + 15 * ((n + 65535) // 65536)


class Stats(C.Structure):
    _fields_ = [
        ("n_files", C.c_uint32), ("n_ok", C.c_uint32), ("n_unsupported", C.c_uint32), ("overflow", C.c_uint32),
        ("in_bytes", C.c_uint64), ("out_bytes", C.c_uint64), ("copy_bytes", C.c_uint64), ("header_bytes", C.c_uint64),
        ("n_tiles", C.c_uint64), ("out_bytes_needed", C.c_uint64),
        ("plan_ms", C.c_float), ("compact_ms", C.c_float), ("h2d_ms", C.c_float), ("d2h_ms", C.c_float),
        ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class TreeStats(C.Structure):
    _fields_ = [
        ("n_selected", C.c_uint32), ("n_gpu", C.c_uint32), ("n_fallback", C.c_uint32), ("n_skipped", C.c_uint32),
        ("n_failed", C.c_uint32), ("n_removed", C.c_uint32),
        ("in_bytes", C.c_uint64), ("out_bytes", C.c_uint64),
        ("walk_read_s", C.c_double), ("gpu_s", C.c_double), ("write_s", C.c_double), ("fallback_s", C.c_double),
        ("read_cpu_s", C.c_double), ("write_cpu_s", C.c_double), ("dma_wait_s", C.c_double), ("io_threads", C.c_uint32), ("n_batches", C.c_uint32),
        ("batch", Stats),
    ]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k != "batch"}
        d["batch"] = self.batch.as_dict()
        return d


class GzipStats(C.Structure):
    _fields_ = [
        ("in_bytes", C.c_uint64), ("out_bytes", C.c_uint64), ("crc32", C.c_uint32), ("n_chunks", C.c_uint32),
        ("n_stored_chunks", C.c_uint32), ("n_fixed_chunks", C.c_uint32), ("deflate_ms", C.c_float), ("crc_ms", C.c_float), ("h2d_ms", C.c_float),
        ("d2h_ms", C.c_float), ("n_opt_chunks", C.c_uint32), ("best_ms", C.c_float),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def zip_bound(n, n_segs):
    """worst-case DEFLATE bytes of one zip piece of n bytes in n_segs segments (LB2_ZIP_BOUND)"""
    return gzip_bound(n) + 17 * n_segs


class ZipSegment(C.Structure):
    _fields_ = [("out_off", C.c_uint64), ("out_len", C.c_uint64), ("crc32", C.c_uint32), ("ended", C.c_uint32)]


class ZipSource(C.Structure):
    _fields_ = [("d_ptr", C.c_void_p), ("len", C.c_uint64)]


class InflateStats(C.Structure):
    _fields_ = [
        ("in_bytes", C.c_uint64), ("out_bytes", C.c_uint64), ("crc32", C.c_uint32), ("n_spans", C.c_uint32),
        ("n_rounds", C.c_uint32), ("n_rejected", C.c_uint32), ("n_absorbed", C.c_uint32),
        ("find_ms", C.c_float), ("count_ms", C.c_float), ("decode_ms", C.c_float), ("resolve_ms", C.c_float),
        ("crc_ms", C.c_float), ("h2d_ms", C.c_float),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class InflateSpan(C.Structure):
    _fields_ = [("in_len", C.c_uint64), ("out_len", C.c_uint64)]


class UnzipMember(C.Structure):
    _fields_ = [("body_off", C.c_uint64), ("body_len", C.c_uint64), ("size", C.c_uint64), ("crc32", C.c_uint32),
                ("method", C.c_uint32)]


class UnzipResult(C.Structure):
    _fields_ = [("out_off", C.c_uint64), ("crc32", C.c_uint32), ("status", C.c_int32)]


class UnzipStats(C.Structure):
    _fields_ = [
        ("in_bytes", C.c_uint64), ("out_bytes", C.c_uint64), ("n_members", C.c_uint32), ("n_stored", C.c_uint32),
        ("n_small", C.c_uint32), ("n_large", C.c_uint32), ("n_spans", C.c_uint32), ("n_rounds", C.c_uint32),
        ("n_rejected", C.c_uint32), ("n_absorbed", C.c_uint32), ("n_bad", C.c_uint32),
        ("h2d_ms", C.c_float), ("copy_ms", C.c_float), ("small_ms", C.c_float), ("find_ms", C.c_float),
        ("count_ms", C.c_float), ("decode_ms", C.c_float), ("resolve_ms", C.c_float), ("crc_ms", C.c_float),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class TarRange(C.Structure):
    _fields_ = [("off", C.c_uint64), ("len", C.c_uint64)]


class TarIndexStats(C.Structure):
    _fields_ = [("n_members", C.c_uint64), ("stop_offset", C.c_uint64), ("stop_reason", C.c_uint32),
                ("kernel_ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class ElfObject(C.Structure):
    _fields_ = [("status", C.c_int32), ("machine", C.c_uint16), ("type", C.c_uint16), ("first_record", C.c_uint32),
                ("n_records", C.c_uint32), ("pool_off", C.c_uint64), ("pool_len", C.c_uint64)]


class ElfRecord(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("flags", C.c_uint32), ("ref", C.c_uint32), ("len", C.c_uint32),
                ("off", C.c_uint64)]


class ElfDepsStats(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("pool_bytes", C.c_uint64), ("bytes_down", C.c_uint64),
                ("kernel_ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SymObject(C.Structure):
    _fields_ = [("status", C.c_int32), ("flags", C.c_uint32), ("nsyms", C.c_uint32), ("nver", C.c_uint32),
                ("nbucket", C.c_uint32), ("symoffset", C.c_uint32), ("bloom_words", C.c_uint32),
                ("bloom_shift", C.c_uint32), ("nrefs", C.c_uint32), ("nhash", C.c_uint32), ("str_len", C.c_uint64),
                ("hash_len", C.c_uint64), ("sym_off", C.c_uint64), ("str_off", C.c_uint64), ("versym_off", C.c_uint64),
                ("hash_off", C.c_uint64), ("rela_off", C.c_uint64), ("rela_n", C.c_uint64), ("plt_off", C.c_uint64),
                ("plt_n", C.c_uint64), ("arena", C.c_uint64), ("refs", C.c_uint64)]


class SymRef(C.Structure):  # elf_syms.cuh Ref: a reference as the arena holds it
    _fields_ = [("sym", C.c_uint32), ("name", C.c_uint32), ("name_len", C.c_uint32), ("gnu", C.c_uint32),
                ("sysv", C.c_uint32), ("ver", C.c_uint16), ("weak", C.c_uint8), ("pad", C.c_uint8)]


class SymJob(C.Structure):
    _fields_ = [("obj", C.c_uint32), ("scope_off", C.c_uint32), ("scope_len", C.c_uint32), ("pad", C.c_uint32)]


class SymMiss(C.Structure):
    _fields_ = [("job", C.c_uint32), ("ref", C.c_uint32)]


class SymQuery(C.Structure):
    _fields_ = [("scope_off", C.c_uint32), ("scope_len", C.c_uint32), ("name_off", C.c_uint32), ("name_len", C.c_uint32)]


class SymFound(C.Structure):
    _fields_ = [("obj", C.c_uint32), ("sym", C.c_uint32), ("info", C.c_uint8), ("other", C.c_uint8),
                ("versym", C.c_uint16)]


class SymsStats(C.Structure):
    _fields_ = [("bytes_up", C.c_uint64), ("bytes_down", C.c_uint64), ("references", C.c_uint64),
                ("lookups", C.c_uint64), ("arena_bytes", C.c_uint64), ("index_ms", C.c_float),
                ("refs_ms", C.c_float), ("resolve_ms", C.c_float), ("pad", C.c_float)]


class FillRegion(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("len", C.c_uint64)]


class NativeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("lambdipy_b200: rc=%d: %s" % (code, msg))
        self.code = code


class NoDeviceError(NativeError):
    pass


_lib = None


def load():
    """dlopen the in-tree CUDA library; raise (never fall back) when it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("%s is missing: run `python -m lambdipy_b200.build` (needs nvcc); "
                          "there is no CPU fallback for the strip path" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, u64p, i32p = C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)
    lib.lb2_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    lib.lb2_ctx_create.restype = C.c_int
    lib.lb2_ctx_destroy.argtypes = [vp]
    lib.lb2_ctx_destroy.restype = None
    lib.lb2_last_error.argtypes = [vp]
    lib.lb2_last_error.restype = C.c_char_p
    lib.lb2_version.restype = C.c_char_p
    lib.lb2_sm_count.argtypes = [vp]
    lib.lb2_sm_count.restype = C.c_int
    lib.lb2_dev_alloc.argtypes = [vp, C.c_uint64]
    lib.lb2_dev_alloc.restype = vp
    lib.lb2_dev_free.argtypes = [vp, vp]
    lib.lb2_dev_free.restype = None
    lib.lb2_pinned_alloc.argtypes = [vp, C.c_uint64]
    lib.lb2_pinned_alloc.restype = vp
    lib.lb2_pinned_free.argtypes = [vp, vp]
    lib.lb2_pinned_free.restype = None
    lib.lb2_memcpy_h2d.argtypes = [vp, vp, vp, C.c_uint64]
    lib.lb2_memcpy_h2d.restype = C.c_int
    lib.lb2_memcpy_d2h.argtypes = [vp, vp, vp, C.c_uint64]
    lib.lb2_memcpy_d2h.restype = C.c_int
    lib.lb2_memset_d.argtypes = [vp, vp, C.c_int, C.c_uint64]
    lib.lb2_memset_d.restype = C.c_int
    lib.lb2_strip_device_async.argtypes = [vp, vp, u64p, u64p, C.c_uint32, vp, C.c_uint64, C.c_uint32, vp]
    lib.lb2_strip_device_async.restype = C.c_int
    lib.lb2_batch_results.argtypes = [vp, u64p, u64p, i32p, C.POINTER(Stats)]
    lib.lb2_batch_results.restype = C.c_int
    lib.lb2_strip_host.argtypes = [vp, vp, u64p, u64p, C.c_uint32, vp, C.c_uint64, u64p, u64p, i32p, C.c_uint32,
                                   C.POINTER(Stats)]
    lib.lb2_strip_host.restype = C.c_int
    lib.lb2_strip_tree.argtypes = [vp, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(TreeStats)]
    lib.lb2_strip_tree.restype = C.c_int
    lib.lb2_plan_device.argtypes = [vp, vp, u64p, u64p, C.c_uint32, C.c_uint32, u64p, i32p, C.POINTER(Stats)]
    lib.lb2_plan_device.restype = C.c_int
    lib.lb2_corpus_fill.argtypes = [vp, vp, C.POINTER(FillRegion), C.c_uint32, C.c_uint64, vp]
    lib.lb2_corpus_fill.restype = C.c_int
    lib.lb2_corpus_scatter.argtypes = [vp, vp, vp, C.c_uint64, u64p, u64p, u64p, C.c_uint32]
    lib.lb2_corpus_scatter.restype = C.c_int
    lib.lb2_strip_device_chunked.argtypes = [vp, vp, u64p, u64p, C.c_uint32, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp,
                                             vp, vp, u64p, i32p, C.POINTER(Stats)]
    lib.lb2_strip_device_chunked.restype = C.c_int
    lib.lb2_strip_tree_ex.argtypes = [vp, C.c_char_p, C.c_char_p, C.c_uint32, C.c_char_p, C.POINTER(TreeStats)]
    lib.lb2_strip_tree_ex.restype = C.c_int
    lib.lb2_tree_cleanup.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(C.c_uint32)]
    lib.lb2_tree_cleanup.restype = C.c_int
    lib.lb2_cleanup_tests_removed.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.c_uint32, C.POINTER(C.c_uint8)]
    lib.lb2_cleanup_tests_removed.restype = C.c_int
    lib.lb2_tree_prepare.argtypes = [vp, C.c_uint64]
    lib.lb2_tree_prepare.restype = C.c_int
    lib.lb2_gzip_create.argtypes = [vp, C.c_uint32, C.POINTER(vp)]
    lib.lb2_gzip_create.restype = C.c_int
    lib.lb2_gzip_submit.argtypes = [vp, vp, C.c_uint64]
    lib.lb2_gzip_submit.restype = C.c_int
    lib.lb2_gzip_collect.argtypes = [vp, vp, C.c_uint64, u64p]
    lib.lb2_gzip_collect.restype = C.c_int
    lib.lb2_gzip_finish.argtypes = [vp, vp, C.c_uint64, u64p, C.POINTER(C.c_uint32), u64p, C.POINTER(GzipStats)]
    lib.lb2_gzip_finish.restype = C.c_int
    lib.lb2_gzip_destroy.argtypes = [vp]
    lib.lb2_gzip_destroy.restype = None
    lib.lb2_inflate_create.argtypes = [vp, C.c_uint32, C.POINTER(vp)]
    lib.lb2_inflate_create.restype = C.c_int
    lib.lb2_inflate_run.argtypes = [vp, vp, C.c_uint64, u64p, C.POINTER(InflateStats)]
    lib.lb2_inflate_run.restype = C.c_int
    lib.lb2_inflate_read.argtypes = [vp, vp, C.c_uint64]
    lib.lb2_inflate_read.restype = C.c_int
    lib.lb2_inflate_destroy.argtypes = [vp]
    lib.lb2_inflate_destroy.restype = None
    lib.lb2_zip_create.argtypes = [vp, C.c_uint32, C.POINTER(vp)]
    lib.lb2_zip_create.restype = C.c_int
    lib.lb2_zip_submit.argtypes = [vp, vp, C.c_uint64, u64p, u64p, C.c_uint32, C.c_uint32]
    lib.lb2_zip_submit.restype = C.c_int
    lib.lb2_zip_submit_device.argtypes = [vp, C.POINTER(ZipSource), C.c_uint32, C.c_uint32]
    lib.lb2_zip_submit_device.restype = C.c_int
    lib.lb2_zip_collect.argtypes = [vp, vp, C.c_uint64, u64p, C.POINTER(ZipSegment), C.POINTER(GzipStats)]
    lib.lb2_zip_collect.restype = C.c_int
    lib.lb2_zip_destroy.argtypes = [vp]
    lib.lb2_zip_destroy.restype = None
    lib.lb2_unzip_create.argtypes = [vp, C.c_uint32, C.POINTER(vp)]
    lib.lb2_unzip_create.restype = C.c_int
    lib.lb2_unzip_run.argtypes = [vp, vp, C.c_uint64, C.POINTER(UnzipMember), C.c_uint32, u64p, C.POINTER(UnzipResult),
                                  C.POINTER(UnzipStats)]
    lib.lb2_unzip_run.restype = C.c_int
    lib.lb2_unzip_read.argtypes = [vp, vp, C.c_uint64]
    lib.lb2_unzip_read.restype = C.c_int
    lib.lb2_unzip_device_output.argtypes = [vp, C.POINTER(vp), u64p]
    lib.lb2_unzip_device_output.restype = C.c_int
    lib.lb2_unzip_destroy.argtypes = [vp]
    lib.lb2_unzip_destroy.restype = None
    lib.lb2_inflate_device_output.argtypes = [vp, C.POINTER(vp), u64p]
    lib.lb2_inflate_device_output.restype = C.c_int
    lib.lb2_memcpy_d2d.argtypes = [vp, vp, vp, C.c_uint64]
    lib.lb2_memcpy_d2d.restype = C.c_int
    lib.lb2_gzip_submit_device.argtypes = [vp, C.POINTER(ZipSource), C.c_uint32]
    lib.lb2_gzip_submit_device.restype = C.c_int
    lib.lb2_tar_index.argtypes = [vp, vp, C.c_uint64, C.POINTER(TarRange), C.c_uint32, C.POINTER(C.c_uint32), vp,
                                  C.c_uint64, u64p, C.POINTER(TarIndexStats)]
    lib.lb2_tar_index.restype = C.c_int
    u32p = C.POINTER(C.c_uint32)
    lib.lb2_gzip_chunk_sizes.argtypes = [vp, u32p, C.c_uint32, u32p]
    lib.lb2_gzip_chunk_sizes.restype = C.c_int
    lib.lb2_inflate_run_table.argtypes = [vp, vp, C.c_uint64, C.POINTER(InflateSpan), C.c_uint32, u64p,
                                          C.POINTER(InflateStats), u32p, u32p]
    lib.lb2_inflate_run_table.restype = C.c_int
    lib.lb2_zip_chunk_sizes.argtypes = [vp, u32p, C.c_uint32, u32p]
    lib.lb2_zip_chunk_sizes.restype = C.c_int
    lib.lb2_unzip_run_table.argtypes = [vp, vp, C.c_uint64, C.POINTER(UnzipMember), C.c_uint32, u32p,
                                        C.POINTER(InflateSpan), u64p, C.POINTER(UnzipResult), C.POINTER(UnzipStats),
                                        u32p, u32p]
    lib.lb2_unzip_run_table.restype = C.c_int
    lib.lb2_elf_deps.argtypes = [vp, u64p, u64p, C.c_uint32, C.POINTER(ElfObject), C.POINTER(ElfRecord), C.c_uint32,
                                 u32p, vp, C.c_uint64, u64p, C.POINTER(ElfDepsStats)]
    lib.lb2_elf_deps.restype = C.c_int
    lib.lb2_syms_create.argtypes = [vp, C.POINTER(vp)]
    lib.lb2_syms_create.restype = C.c_int
    lib.lb2_syms_destroy.argtypes = [vp]
    lib.lb2_syms_destroy.restype = None
    lib.lb2_syms_index.argtypes = [vp, u64p, u64p, C.c_uint32, u32p, C.POINTER(SymObject), C.POINTER(SymsStats)]
    lib.lb2_syms_index.restype = C.c_int
    lib.lb2_syms_resolve.argtypes = [vp, C.POINTER(SymJob), C.c_uint32, u32p, C.c_uint32, C.POINTER(C.c_uint8), u32p,
                                     C.POINTER(SymMiss), C.c_uint32, u32p, C.POINTER(SymsStats)]
    lib.lb2_syms_resolve.restype = C.c_int
    lib.lb2_syms_names.argtypes = [vp, C.POINTER(SymJob), C.c_uint32, C.POINTER(SymMiss), C.c_uint32, u64p, vp,
                                   C.c_uint64, u64p, C.POINTER(SymsStats)]
    lib.lb2_syms_names.restype = C.c_int
    lib.lb2_syms_find.argtypes = [vp, C.POINTER(SymQuery), C.c_uint32, u32p, C.c_uint32, vp, C.c_uint64,
                                  C.POINTER(SymFound), C.POINTER(SymsStats)]
    lib.lb2_syms_find.restype = C.c_int
    _lib = lib
    return lib


# consumer callback of lb2_strip_device_chunked (include/lambdipy_b200.h: lb2_chunk_fn)
CHUNK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64),
                       C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(Stats))


class Context:
    """One CUDA device + the library's workspaces.  Not thread-safe (one per thread and device)."""

    def __init__(self, device=0):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.lb2_ctx_create(int(device), C.byref(h))
        if rc != LB2_OK:
            msg = (self.lib.lb2_last_error(None) or b"").decode()
            raise (NoDeviceError if rc == LB2_E_NODEVICE else NativeError)(rc, msg)
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.lb2_ctx_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc):
        if rc != LB2_OK:
            raise NativeError(rc, (self.lib.lb2_last_error(self.h) or b"").decode())

    @property
    def sm_count(self):
        return self.lib.lb2_sm_count(self.h)

    # -- raw memory helpers -------------------------------------------------------------------
    def dev_alloc(self, n):
        p = self.lib.lb2_dev_alloc(self.h, n)
        if not p:
            raise NativeError(LB2_E_CUDA, (self.lib.lb2_last_error(self.h) or b"").decode())
        return p

    def dev_free(self, p):
        self.lib.lb2_dev_free(self.h, p)

    def pinned_alloc(self, n):
        p = self.lib.lb2_pinned_alloc(self.h, n)
        if not p:
            raise NativeError(LB2_E_CUDA, (self.lib.lb2_last_error(self.h) or b"").decode())
        return p

    def pinned_free(self, p):
        self.lib.lb2_pinned_free(self.h, p)

    def h2d(self, d, h, n):
        self.check(self.lib.lb2_memcpy_h2d(self.h, d, h, n))

    def d2h(self, h, d, n):
        self.check(self.lib.lb2_memcpy_d2h(self.h, h, d, n))

    def d2d(self, dst, src, n):
        self.check(self.lib.lb2_memcpy_d2d(self.h, dst, src, n))
