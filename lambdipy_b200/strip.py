"""Host-side entry points of the CUDA strip path.

`strip_tree(build_directory)` is the call that replaces the reference's shell line
`find {install_dir}/ -name "*.so" | xargs strip` (/root/reference/lambdipy/project_build.py:260);
`strip_buffers` is the same operation on in-memory files (what `xargs` hands to one `strip`).
Every byte of output for status-0 files is produced by the CUDA kernels in csrc/; the only other
executor that can ever touch a file is the host `strip` binary itself -- the reference's own tool --
for ELF classes the device planner reports as unsupported, and only when the caller asks for it.
"""
import ctypes as C
import os

import numpy as np

from . import _native as N

ALIGN = 256


def _round(n, a=ALIGN):
    return (n + a - 1) // a * a


class HostArena:
    """Pinned host memory holding a batch of files at 256-byte aligned offsets."""

    def __init__(self, ctx, sizes):
        self.ctx = ctx
        self.n = len(sizes)
        self.sizes = np.asarray(sizes, dtype=np.uint64)
        off = np.zeros(self.n + 1, dtype=np.uint64)
        if self.n:
            np.cumsum((self.sizes + np.uint64(ALIGN - 1)) // np.uint64(ALIGN) * np.uint64(ALIGN), out=off[1:])
        self.off = off
        self.nbytes = int(off[-1]) + ALIGN
        self.ptr = ctx.pinned_alloc(self.nbytes)
        self.buf = (C.c_uint8 * self.nbytes).from_address(self.ptr)
        self.view = np.frombuffer(self.buf, dtype=np.uint8)

    def put(self, i, data):
        o = int(self.off[i])
        self.view[o:o + len(data)] = np.frombuffer(data, dtype=np.uint8)

    def close(self):
        if self.ptr:
            self.view = None
            self.buf = None
            self.ctx.pinned_free(self.ptr)
            self.ptr = None


def _u64p(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def strip_buffers(ctx, blobs, flags=0, out_slack=None):
    """Strip a list of ELF images (bytes).  Returns (outputs, status, stats):
    outputs[i] is the stripped image for status[i] == 0, else None."""
    n = len(blobs)
    sizes = [len(b) for b in blobs]
    arena = HostArena(ctx, sizes)
    out_cap = arena.nbytes + n * 4096 + (16 << 20) if out_slack is None else arena.nbytes + out_slack
    out_ptr = ctx.pinned_alloc(out_cap)
    try:
        for i, b in enumerate(blobs):
            arena.put(i, b)
        out_off = np.zeros(n + 1, dtype=np.uint64)
        out_sizes = np.zeros(max(n, 1), dtype=np.uint64)
        status = np.zeros(max(n, 1), dtype=np.int32)
        st = N.Stats()
        rc = ctx.lib.lb2_strip_host(ctx.h, arena.ptr, _u64p(arena.off), _u64p(arena.sizes if n else np.zeros(1, np.uint64)), n,
                                    out_ptr, out_cap, _u64p(out_off), _u64p(out_sizes),
                                    status.ctypes.data_as(C.POINTER(C.c_int32)), flags, C.byref(st))
        ctx.check(rc)
        outs = []
        for i in range(n):
            if status[i] == N.ST_OK:
                outs.append(C.string_at(out_ptr + int(out_off[i]), int(out_sizes[i])))
            else:
                outs.append(None)
        return outs, [int(s) for s in status[:n]], st.as_dict()
    finally:
        arena.close()
        ctx.pinned_free(out_ptr)


def strip_tree(root, suffix=".so", device=0, fallback_host_strip=True, tolerate_non_elf=False, dry_run=False, ctx=None,
               cleanup=False, keep_tests_regex=None):
    """Strip every `*{suffix}` regular file under `root` in place.  Returns the tree statistics.

    Selection and side effects follow the reference pipeline (basename match, symlinks and
    directories left alone, new contents written into the existing inode like GNU strip 2.42: mode,
    owner and other hard links kept).  `n_failed > 0` corresponds to the reference script exiting
    non-zero (xargs rc 123).  cleanup=True also performs the script's three `rm -rf` lines
    (/root/reference/lambdipy/project_build.py:256-259) on the same walk; keep_tests_regex is the
    `grep -v` pattern of the `tests` line ("*" when the reference's keep_tests is None)."""
    own = ctx is None
    if own:
        ctx = N.Context(device)
    try:
        flags = 0
        if fallback_host_strip:
            flags |= N.TREE_FALLBACK_HOST_STRIP
        if tolerate_non_elf:
            flags |= N.TREE_TOLERATE_NON_ELF
        if dry_run:
            flags |= N.TREE_DRY_RUN
        if cleanup:
            flags |= N.TREE_CLEANUP
        st = N.TreeStats()
        kr = None if keep_tests_regex is None else os.fsencode(keep_tests_regex)
        ctx.check(ctx.lib.lb2_strip_tree_ex(ctx.h, os.fsencode(root), os.fsencode(suffix), flags, kr, C.byref(st)))
        return st.as_dict()
    finally:
        if own:
            ctx.close()


def cleanup_tree(root, keep_tests_regex="*"):
    """Only the clean-up lines of the reference's script (project_build.py:256-259); needs no GPU."""
    lib = N.load()
    n = C.c_uint32()
    rc = lib.lb2_tree_cleanup(os.fsencode(root), None if keep_tests_regex is None else os.fsencode(keep_tests_regex), C.byref(n))
    if rc != N.LB2_OK:
        raise N.NativeError(rc, "lb2_tree_cleanup(%r)" % root)
    return n.value
