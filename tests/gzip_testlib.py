"""gzip inputs for the tests: a seeded BGZF writer (the member layout `bgzip` writes), plain single-member gzip, concatenated members and
mixed files, and a Python walk over BGZF headers that kmcb200_bgzf_scan is held to.  The compressed bytes depend on the zlib build; the
text they inflate to does not."""
import os
import struct
import zlib

import numpy as np

BGZF_PIECE = 65280                                                      # the text per member bgzip writes (BGZF_BLOCK_SIZE)
BGZF_MAX_TEXT = 65536
# the empty member bgzip ends a file with
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def deflate_raw(text, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem_level=8, flush_every=None, flush_mode=zlib.Z_SYNC_FLUSH):
    """Raw deflate (no header) of text; flush_every: a flush_mode flush after every that many bytes (empty stored blocks in the stream)."""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, mem_level, strategy)
    if not flush_every:
        return c.compress(text) + c.flush()
    out = [c.compress(text[i:i + flush_every]) + c.flush(flush_mode) for i in range(0, len(text), flush_every)]
    return b"".join(out) + c.flush()


_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0] * 8 + [i // 4 for i in range(4, 24)] + [0]
_DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289,
          16385, 24577]
_DEXT = [max(0, i // 2 - 1) for i in range(30)]


def deflate_fixed(tokens):
    """One final fixed-Huffman block of hand-picked tokens: an int is a literal (or any symbol 0..287 as it is coded), a pair is a match
    (length, distance); the end-of-block code is appended.  zlib never emits some legal streams (a distance of 32768) and no malformed ones:
    the tests write those here."""
    acc, n = 3 | (1 << 1), 3                                           # BFINAL = 1, BTYPE = 01

    def put(v, bits):
        nonlocal acc, n
        acc |= v << n
        n += bits

    def code(sym):
        c, bits = (0x30 + sym, 8) if sym < 144 else (0x190 + sym - 144, 9) if sym < 256 else (sym - 256, 7) if sym < 280 else (0xC0 + sym - 280, 8)
        put(int(format(c, "0%db" % bits)[::-1], 2), bits)              # Huffman codes go most significant bit first

    for t in list(tokens) + [256]:
        if isinstance(t, int):
            code(t)
            continue
        length, dist = t
        i = max(j for j in range(29) if _LBASE[j] <= length)
        code(257 + i)
        put(length - _LBASE[i], _LEXT[i])
        d = max(j for j in range(30) if _DBASE[j] <= dist)
        put(int(format(d, "05b")[::-1], 2), 5)
        put(dist - _DBASE[d], _DEXT[d])
    return acc.to_bytes((n + 7) // 8, "little")


def bgzf_member(text, deflated=None, **kw):
    """One BGZF member: the 18-byte header with the BC subfield, the deflate data, CRC32 and ISIZE."""
    data = deflate_raw(text, **kw) if deflated is None else deflated
    head = struct.pack("<BBBBIBBHBBHH", 31, 139, 8, 4, 0, 0, 255, 6, 66, 67, 2, len(data) + 25)
    return head + data + struct.pack("<II", zlib.crc32(text), len(text) & 0xFFFFFFFF)


def bgzf(text, piece=BGZF_PIECE, eof=True, seed=None, **kw):
    """text as BGZF: members of `piece` text bytes (seed: random sizes of 0..piece instead), then the EOF member."""
    rng = np.random.default_rng(seed) if seed is not None else None
    out, pos = [], 0
    while pos < len(text):
        n = piece if rng is None else int(rng.integers(0, piece + 1))
        out.append(bgzf_member(text[pos:pos + n], **kw))
        pos += n
    return b"".join(out) + (BGZF_EOF if eof else b"")


def gzip_single(text, level=6):
    """One plain gzip member (what `gzip` writes): one deflate stream for the whole text."""
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    return c.compress(text) + c.flush()


def gzip_concat(text, parts=3, level=6):
    """Plain gzip members one after the other (`cat a.gz b.gz`)."""
    cut = [len(text) * i // parts for i in range(parts + 1)]
    return b"".join(gzip_single(text[cut[i]:cut[i + 1]], level) for i in range(parts))


def mixed(text, level=6):
    """BGZF for the first half of the text, a plain gzip member for the rest: the reader switches to zlib at the second part."""
    h = len(text) // 2
    return bgzf(text[:h], eof=False, level=level) + gzip_single(text[h:], level)


def inflate_all(raw):
    """zlib over every member of a gzip file: the text the readers must give."""
    out = []
    while raw:
        d = zlib.decompressobj(31)
        out.append(d.decompress(raw))
        if not d.eof:
            raise ValueError("truncated gzip member")
        raw = d.unused_data
    return b"".join(out)


def py_bgzf_scan(raw, capacity, max_members=None):
    """The member walk kmcb200_bgzf_scan makes, restated: (consumed, text_bytes, [(in_off, out_off, in_bytes, isize)]); None when the first
    member is not BGZF."""
    pos = text = 0
    members = []
    while max_members is None or len(members) < max_members:
        h = raw[pos:pos + 18]
        if h[:4] != b"\x1f\x8b\x08\x04"[:len(h[:4])]:
            return None if not members else (pos, text, members)
        if len(h) < 12:
            break
        xlen = struct.unpack("<H", raw[pos + 10:pos + 12])[0]
        if len(raw) - pos < 12 + xlen:
            break
        q, size = 12, None
        while q + 4 <= 12 + xlen:
            slen = struct.unpack("<H", raw[pos + q + 2:pos + q + 4])[0]
            if raw[pos + q:pos + q + 2] == b"BC" and slen == 2 and q + 6 <= 12 + xlen:
                size = struct.unpack("<H", raw[pos + q + 4:pos + q + 6])[0] + 1
                break
            q += 4 + slen
        if size is None or size < 12 + xlen + 10:
            return None if not members else (pos, text, members)
        if size > len(raw) - pos:
            break
        isize = struct.unpack("<I", raw[pos + size - 4:pos + size])[0]
        if isize > BGZF_MAX_TEXT:
            return None if not members else (pos, text, members)
        if isize > capacity - text:
            break
        members.append((pos, text, size, isize))
        pos += size
        text += isize
    return pos, text, members


def write(path, data):
    with open(path, "wb") as f:
        f.write(data)
    return path


def gz_variants(text, level=6):
    """name -> compressed bytes of the same text, one per reader path."""
    return {"bgzf": bgzf(text, level=level), "single": gzip_single(text, level), "concat": gzip_concat(text, 3, level),
            "mixed": mixed(text, level)}


def write_variants(tmp, stem, text, level=6):
    """The plain file and its gzip variants under tmp: {"plain": path, "bgzf": path, ...}."""
    paths = {"plain": write(os.path.join(tmp, stem), text)}
    for name, data in gz_variants(text, level).items():
        paths[name] = write(os.path.join(tmp, "%s.%s.gz" % (stem, name)), data)
    return paths


# ----------------------------------------------------------------------------- the cases of tests/golden/gzip_reference.json
GZIP_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gzip_reference.json")
# name -> (input kind, k, reference options besides -k / the format / -sr1, count_reads keywords)
GZIP_CASES = {
    "fq_k31": ("fq", 31, [], {}),
    "fq_k31_b": ("fq", 31, ["-b"], {"both_strands": False}),
    "fq_k55": ("fq", 55, [], {}),
    "fq_k55_b_n64": ("fq", 55, ["-b", "-n64"], {"both_strands": False, "n_bins": 64}),
    "fq_k31_n64": ("fq", 31, ["-n64"], {"n_bins": 64}),
    "fq_k13_small": ("fq", 13, [], {"small_k": True}),
    "fq_k30_opt_out_size": ("fq", 30, ["--opt-out-size"], {"opt_out_size": True}),
    "fq_k31_hc": ("fq", 31, ["-hc"], {"homopolymer_compressed": True}),
    "fa_k31": ("fa", 31, [], {}),
    "fm_k31": ("fm", 31, [], {}),
    "fq_k31_e": ("fq", 31, ["-e"], {}),
}
FORMAT_FLAG = {"fq": "-fq", "fa": "-fa", "fm": "-fm"}


def case_text(kind):
    """The seeded text of a case input: 12,000 reads of 150 bases (FASTQ, one-line FASTA) or 1,500 reads of 1,200 (60-base lines)."""
    from stage1_testlib import make_reads
    if kind == "fq":
        reads = make_reads(2031, "short", n_reads=12000)
        return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)) for i, r in enumerate(reads))
    if kind == "fa":
        reads = make_reads(2032, "short", n_reads=12000)
        return b"".join(b">r%d\n%s\n" % (i, r) for i, r in enumerate(reads))
    reads = make_reads(2033, "short", n_reads=1500, read_len=1200)
    return b"".join(b">r%d\n" % i + b"\n".join(r[j:j + 60] for j in range(0, len(r), 60)) + b"\n" for i, r in enumerate(reads))
