"""Seeded mutants of a shared object for the bounds checks of the dynamic-section parse (elf_deps.cuh): header fields,
program-header offsets and sizes, dynamic values past the end, version-chain links and counts (a next link of 0 loops
on its own entry; counts up to 2^32), strings cut at EOF and string tables without a NUL, and random flips in the
headers.  Test data only."""
import random
import struct

def mutants(data, seed):
    """yield (label, bytes)"""
    rnd = random.Random(seed)
    b = bytes(data)
    phoff, = struct.unpack_from("<Q", b, 32); phnum, = struct.unpack_from("<H", b, 56)
    big = [len(b), len(b) - 1, len(b) + 1, 1 << 32, (1 << 64) - 1, (1 << 63), rnd.randrange(1 << 64)]
    def put(fmt, off, v):
        m = bytearray(b); struct.pack_into(fmt, m, off, v & ((1 << (8*struct.calcsize(fmt))) - 1)); return bytes(m)
    for v in (0, 1, 3, 0xffff, rnd.randrange(1 << 16)):
        yield "e_phnum=%d" % v, put("<H", 56, v)
    for v in big + [0, 1]:
        yield "e_phoff=%d" % v, put("<Q", 32, v)
    yield "e_phentsize=32", put("<H", 54, 32)
    yield "class=1", put("<B", 4, 1); yield "data=2", put("<B", 5, 2); yield "class=9", put("<B", 4, 9)
    dyn = None
    for i in range(phnum):
        t, = struct.unpack_from("<I", b, phoff + 56*i)
        if t in (1, 2):
            for f, name in ((8, "p_offset"), (16, "p_vaddr"), (32, "p_filesz")):
                for v in big[:5]:
                    yield "ph%d.%s=%x" % (i, name, v), put("<Q", phoff + 56*i + f, v)
        if t == 2: dyn = struct.unpack_from("<QQQQQ", b, phoff + 56*i + 8)
    if dyn:
        off, va, pa, fsz, msz = dyn
        ents = [(off + 16*k, *struct.unpack_from("<qQ", b, off + 16*k)) for k in range(fsz // 16)]
        for at, tag, val in ents:
            if tag in (1, 5, 10, 14, 15, 29, 0x6ffffffc, 0x6ffffffd, 0x6ffffffe, 0x6fffffff):
                for v in big + [val + 1, val - 1, 0]:
                    yield "d_val[%x]=%x" % (tag, v), put("<Q", at + 8, v)
            if tag == 0:
                break
        # chains: vn_next / vna_next / vd_next mutated in place where the section starts
        def vaddr2off(a):
            for i in range(phnum):
                t, fl, po, pv, pp, fs = struct.unpack_from("<IIQQQQ", b, phoff + 56*i)
                if t == 1 and pv <= a < pv + fs: return a - pv + po
        tags = {tag: val for _, tag, val in ents}
        for tag, fields in ((0x6ffffffe, (2, 4, 8, 12)), (0x6ffffffc, (6, 12, 16))):
            if tag in tags:
                o = vaddr2off(tags[tag])
                for f in fields:
                    for v in (0, 1, 15, 0xffff, 0xffffffff, rnd.randrange(1 << 16)):
                        fmt = "<H" if f in (2, 6) else "<I"
                        yield "chain[%x]+%d=%x" % (tag, f, v), put(fmt, o + f, v)
                # the first Vernaux / Verdaux link
                if tag == 0x6ffffffe:
                    aux = o + struct.unpack_from("<I", b, o + 8)[0]
                    for v in (0, 16, 0xffffffff): yield "vna_next=%x" % v, put("<I", aux + 12, v)
                    for v in (0, 0xffffffff, len(b)): yield "vna_name=%x" % v, put("<I", aux + 8, v)
        # strings cut at EOF: the file ends inside .dynstr
        if 5 in tags:
            s0 = vaddr2off(tags[5])
            for cut in (s0 + 1, s0 + 10, s0 + tags.get(10, 0) // 2, s0 + tags.get(10, 1) - 1):
                if 0 < cut < len(b): yield "cut@%d" % cut, b[:cut]
            # a string table without a NUL to its end
            m = bytearray(b); sz = tags.get(10, 0)
            for k in range(s0, min(s0 + sz, len(b))):
                if m[k] == 0: m[k] = 0x41
            yield "no_nul", bytes(m)
    for _ in range(20):  # random byte flips in the header and program headers
        m = bytearray(b)
        for _ in range(3):
            k = rnd.randrange(min(len(b), phoff + 56 * max(phnum, 1)))
            m[k] = rnd.randrange(256)
        yield "flip", bytes(m)
