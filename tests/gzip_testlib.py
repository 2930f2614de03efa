"""gzip inputs for the tests: a seeded BGZF writer (the member layout `bgzip` writes), plain single-member gzip, concatenated members and
mixed files, and a Python walk over BGZF headers that kmcb200_bgzf_scan is held to.  The compressed bytes depend on the zlib build; the
text they inflate to does not."""
import os
import struct
import zlib

import numpy as np

BGZF_PIECE = 65280                                                      # the text per member bgzip writes (BGZF_BLOCK_SIZE)
BGZF_MAX_TEXT = 65536
BGZF_MAX_DATA = 65536 - 26                                              # the deflate data of a member: BSIZE < 2^16, 18 + 8 bytes of frame
# the empty member bgzip ends a file with
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def deflate_raw(text, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem_level=8, flush_every=None, flush_mode=zlib.Z_SYNC_FLUSH):
    """Raw deflate (no header) of text; flush_every: a flush_mode flush after every that many bytes (empty stored blocks in the stream)."""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, mem_level, strategy)
    if not flush_every:
        return c.compress(text) + c.flush()
    out = [c.compress(text[i:i + flush_every]) + c.flush(flush_mode) for i in range(0, len(text), flush_every)]
    return b"".join(out) + c.flush()


# ----------------------------------------------------------------------------- a DEFLATE writer (RFC 1951) for the streams zlib never writes
# zlib's deflate writes one habit of the format: both trees run-length coded apart, at least two distance codes, no empty trees, HLIT /
# HDIST / HCLEN no larger than needed.  Other encoders (libdeflate behind bgzip and samtools, other gzip writers) write other legal shapes,
# and no encoder writes malformed ones.  This writer puts every field of a block under the caller's control.
_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0] * 8 + [i // 4 for i in range(4, 24)] + [0]
_DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289,
          16385, 24577]
_DEXT = [max(0, i // 2 - 1) for i in range(30)]
CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT_LENS = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST_LENS = [5] * 32
_LSYM = [0] * 3 + [max(j for j in range(29) if _LBASE[j] <= n) for n in range(3, 259)]   # length -> symbol - 257 (258: 285)


class Match:
    """A match token written with a chosen length symbol (257..287) and distance symbol (0..31) and their extra bits: Match(284, 31, d, e)
    is length 258 the long way.  A pair (length, distance) is a match with the usual symbols."""
    __slots__ = ("lsym", "lextra", "dsym", "dextra")

    def __init__(self, lsym, lextra, dsym, dextra):
        self.lsym, self.lextra, self.dsym, self.dextra = lsym, lextra, dsym, dextra

    @staticmethod
    def of(length, dist):
        ls = _LSYM[length]
        ds = max(j for j in range(30) if _DBASE[j] <= dist)
        return Match(257 + ls, length - _LBASE[ls], ds, dist - _DBASE[ds])

    def length(self):
        return _LBASE[self.lsym - 257] + self.lextra

    def dist(self):
        return _DBASE[self.dsym] + self.dextra


class Bits:
    """n raw bits, least significant first: as a token, any code (one with no symbol too); as a block, anything between blocks."""
    __slots__ = ("value", "n")

    def __init__(self, value, n):
        self.value, self.n = value, n


class Stored:
    """A stored block of `data` (LEN = len(data), up to 65535); bad_nlen: NLEN is not LEN's complement.  final=None: final when last."""

    def __init__(self, data, final=None, bad_nlen=False):
        self.data, self.final, self.bad_nlen = bytes(data), final, bad_nlen


class Fixed:
    """A fixed-Huffman block of tokens: an int is a symbol 0..287 as it is coded (a literal below 256), a pair (length, distance) or a Match
    is a match, a Bits is written as it is; the end-of-block code follows unless eob is False."""

    def __init__(self, tokens, final=None, eob=True):
        self.tokens, self.final, self.eob = list(tokens), final, eob


class Dynamic:
    """A dynamic-Huffman block of tokens (as Fixed's).  The code lengths default to a length-limited Huffman code of the tokens' symbol counts
    (`limit` bits; an empty distance tree when no match uses one); lit_lens / dist_lens give them explicitly, complete or not.  hlit / hdist
    / hclen default to what the lengths need and may be set above it (hlit up to 288, hdist up to 32).  rle: how the lengths are coded,
    "plain" (one symbol each), "runs" (16 / 17 / 18 runs in each tree apart, as zlib does) or "cross" (runs over both trees, so a run may
    cross from the literal/length lengths into the distance ones); cl_syms: the code-length symbols themselves, an int 0..15 or a pair
    (16 | 17 | 18, repeat count).  cl_lens: the code-length code's 19 lengths by symbol (default: a Huffman code limited to 7 bits)."""

    def __init__(self, tokens=(), lit_lens=None, dist_lens=None, hlit=None, hdist=None, hclen=None, rle="runs", cl_syms=None, cl_lens=None,
                 final=None, eob=True, limit=15):
        self.tokens, self.lit_lens, self.dist_lens = list(tokens), lit_lens, dist_lens
        self.hlit, self.hdist, self.hclen, self.rle, self.cl_syms, self.cl_lens = hlit, hdist, hclen, rle, cl_syms, cl_lens
        self.final, self.eob, self.limit = final, eob, limit

    def code_lengths(self):
        """(literal/length lengths padded to HLIT, distance lengths padded to HDIST, HLIT, HDIST) as the block writes them."""
        lit, dist = self.lit_lens, self.dist_lens
        if lit is None or dist is None:
            lf, df = [0] * 286, [0] * 30
            for t in self.tokens:
                if isinstance(t, int):
                    lf[t] += 1
                elif not isinstance(t, Bits):
                    m = t if isinstance(t, Match) else Match.of(*t)
                    lf[m.lsym] += 1
                    df[m.dsym] += 1
            if self.eob:
                lf[256] += 1
            lit = huffman_lengths(lf, self.limit) if lit is None else lit
            dist = huffman_lengths(df, self.limit) if dist is None else dist
        lit, dist = list(lit), list(dist)
        hlit = self.hlit or max(257, max((i + 1 for i, v in enumerate(lit) if v), default=0))
        hdist = self.hdist or max(1, max((i + 1 for i, v in enumerate(dist) if v), default=0))
        return (lit + [0] * hlit)[:hlit], (dist + [0] * hdist)[:hdist], hlit, hdist


def huffman_lengths(freq, limit):
    """Code lengths of a Huffman code for the symbol counts `freq`, no code longer than `limit` bits (the deepest leaves are moved up in
    pairs, which keeps the code complete); a lone symbol gets one 1-bit code, no symbol no code."""
    import heapq
    syms = [s for s, f in enumerate(freq) if f]
    lens = [0] * len(freq)
    if len(syms) < 2:
        for s in syms:
            lens[s] = 1
        return lens
    assert len(syms) <= 1 << limit
    heap = [(freq[s], k) for k, s in enumerate(syms)]
    heapq.heapify(heap)
    parent = [0] * (2 * len(syms) - 1)
    nxt = len(syms)
    while len(heap) > 1:
        f1, a = heapq.heappop(heap)
        f2, b = heapq.heappop(heap)
        parent[a] = parent[b] = nxt
        heapq.heappush(heap, (f1 + f2, nxt))
        nxt += 1
    depth = [0] * nxt
    for k in range(nxt - 2, -1, -1):
        depth[k] = depth[parent[k]] + 1
    count = [0] * (max(depth[:len(syms)]) + 1)
    for k in range(len(syms)):
        count[depth[k]] += 1
    for i in range(len(count) - 1, limit, -1):                         # JPEG's Annex K.3 length limiting
        while count[i] > 0:
            j = i - 2
            while count[j] == 0:
                j -= 1
            count[i] -= 2
            count[i - 1] += 1
            count[j + 1] += 2
            count[j] -= 1
    order = sorted(syms, key=lambda s: (-freq[s], s))
    k = 0
    for length in range(1, min(limit, len(count) - 1) + 1):
        for _ in range(count[length]):
            lens[order[k]] = length
            k += 1
    return lens


def canonical_codes(lens):
    """RFC 1951 §3.2.2: the canonical code of every symbol as (bits reversed for writing, length), None for length 0.  Over-subscribed
    lengths get codes too (cut to their length), so malformed trees can be written."""
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for n in lens:
        if not n:
            out.append(None)
            continue
        c = nxt[n] & ((1 << n) - 1)
        nxt[n] += 1
        out.append((int(format(c, "0%db" % n)[::-1], 2), n))          # Huffman codes go most significant bit first
    return out


def rle_lengths(seq, hlit, mode):
    """The code-length symbols of seq (the HLIT literal/length lengths, then the distance ones): see Dynamic's rle."""
    if mode == "plain":
        return list(seq)
    out = []
    for part in ([seq] if mode == "cross" else [seq[:hlit], seq[hlit:]]):
        i = 0
        while i < len(part):
            v, j = part[i], i
            while j < len(part) and part[j] == v:
                j += 1
            run = j - i
            if v == 0:
                while run >= 11:
                    out.append((18, min(run, 138)))
                    run -= out[-1][1]
                if run >= 3:
                    out.append((17, run))
                    run = 0
            else:
                out.append(v)
                run -= 1
                while run >= 3:
                    out.append((16, min(run, 6)))
                    run -= out[-1][1]
            out += [v] * run
            i = j
    return out


class _BitWriter:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def pos(self):
        return len(self.out) * 8 + self.n


def _put_tokens(w, tokens, lcodes, dcodes):
    for t in tokens:
        if isinstance(t, Bits):
            w.put(t.value, t.n)
            continue
        if isinstance(t, int):
            if lcodes[t] is None:
                raise ValueError("symbol %d has no code" % t)
            w.put(*lcodes[t])
            continue
        m = t if isinstance(t, Match) else Match.of(*t)
        if lcodes[m.lsym] is None or dcodes[m.dsym] is None:
            raise ValueError("match symbols %d / %d have no code" % (m.lsym, m.dsym))
        w.put(*lcodes[m.lsym])
        w.put(m.lextra, _LEXT[m.lsym - 257] if m.lsym < 286 else 0)
        w.put(*dcodes[m.dsym])
        w.put(m.dextra, _DEXT[m.dsym] if m.dsym < 30 else 0)


_FIXED_CODES = (canonical_codes(FIXED_LIT_LENS), canonical_codes(FIXED_DIST_LENS))


def deflate(blocks, seed=None, layout=None):
    """Raw DEFLATE of a list of Stored / Fixed / Dynamic blocks (and Bits between them).  seed: the bits that pad a stored block's header
    to a byte and the final byte are random (decoders ignore them), else 0.  layout: a list that gets (header bit, first data bit, end bit)
    per block."""
    import random
    rng = random.Random(seed) if seed is not None else None
    w = _BitWriter()
    for i, b in enumerate(blocks):
        start = w.pos()
        if isinstance(b, Bits):
            w.put(b.value, b.n)
            continue
        w.put(int(i == len(blocks) - 1 if b.final is None else b.final), 1)
        if isinstance(b, Stored):
            w.put(0, 2)
            pad = -w.pos() % 8
            w.put(rng.getrandbits(pad) if rng and pad else 0, pad)
            n = len(b.data)
            w.put(n, 16)
            w.put(~n & 0xFFFF ^ (0x0100 if b.bad_nlen else 0), 16)
            data = w.pos()
            w.out += b.data
        elif isinstance(b, Fixed):
            w.put(1, 2)
            data = w.pos()
            _put_tokens(w, b.tokens + ([256] if b.eob else []), *_FIXED_CODES)
        else:
            lit, dist, hlit, hdist = b.code_lengths()
            cl_syms = b.cl_syms if b.cl_syms is not None else rle_lengths(lit + dist, hlit, b.rle)
            cl_lens = b.cl_lens
            if cl_lens is None:
                cf = [0] * 19
                for s in cl_syms:
                    cf[s if isinstance(s, int) else s[0]] += 1
                cl_lens = huffman_lengths(cf, 7)
            hclen = b.hclen or max(4, max(i + 1 for i, s in enumerate(CLORDER) if cl_lens[s]))
            w.put(2, 2)
            w.put(hlit - 257, 5)
            w.put(hdist - 1, 5)
            w.put(hclen - 4, 4)
            for s in CLORDER[:hclen]:
                w.put(cl_lens[s], 3)
            ccodes = canonical_codes(cl_lens)
            for s in cl_syms:
                sym, rep = (s, 0) if isinstance(s, int) else s
                w.put(*ccodes[sym])
                if sym >= 16:
                    w.put(rep - (11 if sym == 18 else 3), (2, 3, 7)[sym - 16])
            data = w.pos()
            _put_tokens(w, b.tokens + ([256] if b.eob else []), canonical_codes(lit + [0] * 2), canonical_codes(dist + [0] * 2))
        if layout is not None:
            layout.append((start, data, w.pos()))
    pad = -w.pos() % 8
    w.put(rng.getrandbits(pad) if rng and pad else 0, pad)
    return bytes(w.out)


def spell(tokens, out=None):
    """The text a block's tokens stand for (appended to out, the text before the block, which matches may reach into)."""
    out = bytearray() if out is None else out
    for t in tokens:
        if isinstance(t, int):
            if t >= 256:
                raise ValueError("symbol %d is no literal" % t)
            out.append(t)
            continue
        if isinstance(t, Bits):
            raise ValueError("raw bits have no text")
        length, dist = (t.length(), t.dist()) if isinstance(t, Match) else t
        if not 0 < dist <= len(out):
            raise ValueError("distance %d before the start" % dist)
        start = len(out) - dist
        while length > 0:
            n = min(length, dist)
            out += out[start:start + n]
            start += n
            length -= n
    return out


def blocks_text(blocks):
    """The text a list of blocks inflates to."""
    out = bytearray()
    for b in blocks:
        if isinstance(b, Stored):
            out += b.data
        elif not isinstance(b, Bits):
            spell(b.tokens, out)
    return bytes(out)


# ----------------------------------------------------------------------------- zlib as the oracle of a deflate stream
# the kernel's error codes (inflate.cuh, the low byte of the error word) and the reasons gz_error_name gives them
GZ_ERRORS = {
    "member": (1, "not a BGZF member inside the buffer (header, sizes or output slice)"),
    "block_type": (2, "invalid block type"),
    "stored": (3, "stored block length does not match its complement"),
    "code_set": (4, "over-subscribed or incomplete code set"),
    "code": (5, "invalid literal/length or distance code"),
    "distance": (6, "distance too far back"),
    "output": (7, "more output than the member's ISIZE"),
    "truncated": (8, "deflate data ends before its final block"),
    "isize": (9, "ISIZE does not match the inflated length"),
    "crc": (10, "CRC32 mismatch"),
    "trailing": (11, "bytes between the deflate stream and the trailer"),
    "repeat": (12, "invalid code-length repeat"),
    "no_eob": (13, "no end-of-block code"),
}
# zlib's verdict on a deflate stream -> the kernel's error: its messages, "unfinished" (no error, not at the end) and "trailing" (bytes
# after the end)
ZLIB_TO_KERNEL = {
    "invalid code lengths set": "code_set",
    "invalid literal/lengths set": "code_set",
    "invalid distances set": "code_set",
    "too many length or distance symbols": "code_set",
    "invalid bit length repeat": "repeat",
    "invalid code -- missing end-of-block": "no_eob",
    "invalid literal/length code": "code",
    "invalid distance code": "code",
    "invalid distance too far back": "distance",
    "invalid block type": "block_type",
    "invalid stored block lengths": "stored",
    "unfinished": "truncated",
    "trailing": "trailing",
}


def zlib_inflate(data, limit=BGZF_MAX_TEXT):
    """zlib's verdict on raw deflate data: ("ok", text), ("error", message), ("unfinished", text so far), ("trailing", text) when bytes
    follow the end, or ("oversize", None) past `limit` bytes of text."""
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(data, limit + 1)
    except zlib.error as e:
        return "error", str(e).split(": ", 1)[-1]
    if len(out) > limit:
        return "oversize", None
    if not d.eof:
        return "unfinished", out
    return ("trailing" if d.unused_data else "ok"), out


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


# ----------------------------------------------------------------------------- named streams zlib never writes, valid and malformed
def _fq_source(seed):
    from test_fastx_model import fastq_text
    return fastq_text(seed, 2000, max_len=150)


def random_tokens(rng, size, literal, pos0=0, match_rate=0.3, lsyms=range(257, 286), dsyms=range(30), dist_max=32768):
    """Tokens of at most `size` text bytes after pos0 bytes of text: literals from literal() and, at match_rate, matches whose length and
    distance symbols are drawn from lsyms / dsyms with random extra bits (distances only as far back as the text goes)."""
    lsyms, dsyms = list(lsyms), list(dsyms)
    toks, n = [], 0
    while n < size:
        at = pos0 + n
        if at and dsyms and lsyms and rng.random() < match_rate:
            ls = rng.choice(lsyms)
            le = rng.randrange(1 << _LEXT[ls - 257])
            ds = rng.choice(dsyms)
            if _DBASE[ds] <= min(at, dist_max) and n + _LBASE[ls - 257] + le <= size:
                de = rng.randrange(min(1 << _DEXT[ds], min(at, dist_max) - _DBASE[ds] + 1))
                toks.append(Match(ls, le, ds, de))
                n += _LBASE[ls - 257] + le
                continue
        toks.append(literal())
        n += 1
    return toks


def _lit_from(rng, alphabet):
    return lambda: alphabet[rng.randrange(len(alphabet))]


def _lit_seq(text, start=0):
    it = iter(text[start:] + text)
    return lambda: next(it)


def _lens(spec, n):
    """Code lengths from {symbol or range: length}."""
    out = [0] * n
    for k, v in spec.items():
        for s in (k if isinstance(k, range) else [k]):
            out[s] = v
    return out


def shape_blocks():
    """name -> (blocks, seed): valid stream shapes that zlib's deflate never writes, each decoded by zlib (tests/test_gzip_model.py)."""
    import random
    rng = random.Random(7001)
    fq = _fq_source(7002)
    big = 60_000
    s = {}
    # a 16 run from the last literal/length lengths (226..285: 9 bits) into the distance lengths (0..3: 9 bits, the 9-bit distance codes)
    lit = _lens({range(0, 226): 8, range(226, 286): 9}, 286)
    dist = [9, 9, 9, 9, 1, 2, 3, 4, 5, 6, 7]
    s["repeat16_across_trees"] = [Dynamic(random_tokens(rng, big, _lit_from(rng, range(256)), dsyms=range(11)), lit, dist, rle="cross")]
    # an 18 run of zeros from the literal/length lengths (280..285) into the distance lengths (0..4)
    lit = _lens({range(0, 232): 8, range(232, 280): 9}, 286)
    dist = _lens({range(5, 12): 4, range(12, 30): 5}, 30)
    s["zero_run_across_trees"] = [Dynamic(random_tokens(rng, big, _lit_from(rng, range(256)), lsyms=range(257, 280), dsyms=range(5, 30)),
                                          lit, dist, hlit=286, rle="cross")]
    # distance trees of one 1-bit code: distance symbol 0 (distance 1), then symbol 9 (25..32)
    t1 = random_tokens(rng, 30_000, _lit_seq(fq), dsyms=[0])
    t2 = random_tokens(rng, 30_000, _lit_seq(fq, 500), pos0=len(spell(t1)), dsyms=[9])
    s["single_1bit_distance_code"] = [Dynamic(t1, dist_lens=[1]), Dynamic(t2, dist_lens=_lens({9: 1}, 10))]
    # a literal/length tree that is one 1-bit end-of-block code (an empty block), between and after other blocks
    eob_only = dict(lit_lens=_lens({256: 1}, 257), dist_lens=[0])
    s["single_1bit_end_of_block"] = [Dynamic(**eob_only), Fixed(fq[:5000]), Dynamic(**eob_only), Dynamic(**eob_only)]
    # literal-only dynamic blocks without distance codes: HDIST 1 with length 0, and HDIST 30 all 0
    s["literal_only_empty_distance_tree"] = [Dynamic(fq[:30_000], dist_lens=[0]), Dynamic(fq[30_000:big], dist_lens=[0] * 30, hdist=30)]
    # header extremes: HLIT 257 / HDIST 1 (literals, one unused distance code), HLIT 286 / HDIST 30 with every length and distance symbol in use,
    # and HLIT 286 / HDIST 30 above what literal-only lengths need
    s["hlit_257_hdist_1"] = [Dynamic(fq[:20_000], dist_lens=[1])]
    s["hlit_286_hdist_30"] = [Dynamic(random_tokens(rng, big, _lit_from(rng, b"ACGT\n"), match_rate=0.5))]
    s["hlit_hdist_above_need"] = [Dynamic(fq[:20_000], hlit=286, hdist=30)]
    assert s["hlit_286_hdist_30"][0].code_lengths()[2:] == (286, 30)
    # HCLEN 5..19, one block each: 255 literals and end-of-block at 8 bits need the code-length symbols 0, 8 and 16 (HCLEN 5) only
    lit8 = _lens({range(0, 255): 8, 256: 8}, 257)
    s["hclen_5_to_19"] = [Dynamic([rng.randrange(255) for _ in range(3000)], lit8, [0], hclen=h) for h in range(5, 20)]
    # distance codes of 1..15 bits (9..15 take the bit-by-bit path past the 8-bit lookup), every one used many times
    dist = list(range(1, 16)) + [15]
    s["distance_codes_9_to_15_bits"] = [Dynamic(random_tokens(rng, big, _lit_seq(fq), match_rate=0.6, lsyms=range(257, 265), dsyms=range(16)),
                                                 dist_lens=dist)]
    # literal/length codes of exactly 10 bits (the last the lookup holds: literals 248..255, end-of-block, lengths 257..277) and 11 bits
    # (the first it does not: lengths 278..281)
    lit = _lens({range(0, 248): 8, range(248, 278): 10, range(278, 282): 11}, 282)
    s["literal_codes_10_and_11_bits"] = [Dynamic(random_tokens(rng, big, _lit_from(rng, range(256)), match_rate=0.4, lsyms=range(257, 282)),
                                                 lit_lens=lit)]
    # stored, fixed and dynamic blocks in one member, a stored block (LEN 0 among them) at each of the 8 bit phases
    mixed, at = [], 0
    for phase in range(8):
        deflate(mixed + [Stored(b"", final=False)], layout=(lay := []))
        cur = lay[-1][0] if lay else 0
        k = (phase - cur - 10) % 8
        mixed.append(Fixed([200] * k + list(fq[at:at + 300])))          # literal 200: 9 bits; header + end-of-block: 10
        mixed.append(Stored(fq[at + 300:at + 300 + 97 * phase]))
        mixed.append(Dynamic(random_tokens(rng, 2000, _lit_seq(fq, at), pos0=len(blocks_text(mixed)))))
        at += 3000
    s["mixed_blocks_stored_every_phase"] = mixed
    s["stored_largest"] = [Stored(fq[:BGZF_MAX_DATA - 5])]                 # the largest stored block a BGZF member holds
    # length 258 as symbol 284 with extra bits 31, in a fixed and a dynamic block
    t = list(fq[:2000]) + [Match(284, 31, 3, 0), Match(284, 31, 10, 5)] * 20 + list(fq[2000:4000]) + [(258, 1)] * 5
    s["length_258_as_284_31"] = [Fixed(t, final=False), Dynamic(t[:len(t) // 2] + [Match(284, 31, 0, 0)] * 50)]
    return {k: (v, 7100 + i) for i, (k, v) in enumerate(sorted(s.items()))}


def shape_streams():
    """name -> (deflate data, text) of shape_blocks()."""
    return {k: (deflate(b, seed=sd), blocks_text(b)) for k, (b, sd) in shape_blocks().items()}


def malformed_streams():
    """name -> (deflate data, text the member's trailer is framed with, the kernel's error (GZ_ERRORS)): one case per validation rule that
    a deflate stream can break.  zlib refuses each for the reason ZLIB_TO_KERNEL maps to the same error (tests/test_gzip_model.py)."""
    t = list(b"ACGTTGCA\n" * 20)
    text = bytes(t)
    good = Dynamic(t)
    lit, dist, hlit, hdist = good.code_lengths()
    cl = rle_lengths(lit + dist, hlit, "runs")
    cf = [0] * 19
    for x in cl:
        cf[x if isinstance(x, int) else x[0]] += 1
    cl_lens = huffman_lengths(cf, 7)
    longest = max(range(19), key=lambda s: (cl_lens[s], s))
    cl_incomplete = cl_lens[:]
    cl_incomplete[longest] += 1
    shortest = min((s for s in range(19) if cl_lens[s]), key=lambda s: (cl_lens[s], s))
    cl_over = cl_lens[:]
    cl_over[shortest] -= 1
    lit_ab = _lens({97: 1, 98: 1}, 257)
    tm = t[:9] + [(9, 9)]                                               # a match at distance symbol 6
    tm_text = bytes(spell(tm))
    lit_m = huffman_lengths([1] * 286, 15)                              # every literal/length symbol
    m = {
        "block_type_3": ([Bits(7, 11)], b"", "block_type"),                # two bytes: the shortest deflate data of a BGZF member
        "stored_length": ([Stored(b"ab", bad_nlen=True)], b"ab", "stored"),
        "stored_length_past_data": (bytes.fromhex("01000100006162"), b"ab", "stored"),    # LEN 256 is past the data, NLEN wrong
        "stored_truncated": (deflate([Stored(text * 10)])[:-100], text * 10, "truncated"),
        "no_final_block": ([Fixed(t, final=False)], text, "truncated"),
        "truncated_dynamic_header": (deflate([good])[:20], text, "truncated"),
        "trailing_byte": (deflate([good]) + b"\x00", text, "trailing"),
        "oversubscribed_literal_set": ([Dynamic(t, lit_lens=_lens({range(0, 257): 8}, 257))], text, "code_set"),
        "oversubscribed_distance_set": ([Dynamic(tm, dist_lens=_lens({0: 1, 1: 1, 6: 1}, 7))], tm_text, "code_set"),
        "incomplete_literal_set": ([Dynamic([97], lit_lens=_lens({97: 2, 256: 2}, 257))], b"a", "code_set"),
        "incomplete_distance_set": ([Dynamic(tm, dist_lens=_lens({0: 2, 6: 2}, 7))], tm_text, "code_set"),
        "lone_2bit_end_of_block": ([Dynamic([], lit_lens=_lens({256: 2}, 257), dist_lens=[0])], b"", "code_set"),
        "lone_2bit_distance_code": ([Dynamic(tm, dist_lens=_lens({6: 2}, 7))], tm_text, "code_set"),
        "incomplete_code_length_code": ([Dynamic(t, cl_lens=cl_incomplete)], text, "code_set"),
        "oversubscribed_code_length_code": ([Dynamic(t, cl_lens=cl_over)], text, "code_set"),
        "hlit_287": ([Dynamic(t, hlit=287)], text, "code_set"),
        "hlit_288": ([Dynamic(t, hlit=288)], text, "code_set"),
        "hlit_287_at_data_end": (deflate([Dynamic(t, hlit=287)])[:3], text, "code_set"),  # the data ends where HCLEN's lengths begin
        "hdist_31": ([Dynamic(t, hdist=31)], text, "code_set"),
        "hdist_32": ([Dynamic(t, hdist=32)], text, "code_set"),
        "repeat16_without_previous": ([Dynamic(t, cl_syms=[(16, 3)] + lit + dist)], text, "repeat"),
        "repeat16_past_end": ([Dynamic(t, cl_syms=lit + dist[:-2] + [(16, 3)])], text, "repeat"),
        "repeat17_past_end": ([Dynamic(t, cl_syms=lit + dist[:-2] + [(17, 3)])], text, "repeat"),
        "repeat18_past_end": ([Dynamic(t, cl_syms=lit[:-5] + [(18, 11)])], text, "repeat"),
        "no_end_of_block": ([Dynamic([97, 98], lit_lens=lit_ab, dist_lens=[0], eob=False)], b"ab", "no_eob"),
        "empty_code_length_code": ([Dynamic([], lit_lens=[0] * 257, dist_lens=[0], cl_syms=[], cl_lens=[0] * 19, hclen=4, eob=False),
                                    Bits(0, 258)], b"", "no_eob"),       # zlib reads each length as 0, one bit each
        "hclen_4": ([Dynamic([], lit_lens=[0] * 257, dist_lens=[0], cl_lens=_lens({18: 1, 0: 1}, 19), eob=False)], b"", "no_eob"),
        "invalid_code": ([Fixed([97, 286])], b"aaaa", "code"),
        "invalid_code_287": ([Fixed([97, 287])], b"aaaa", "code"),
        "invalid_distance_code_30": ([Fixed([97, Match(257, 0, 30, 0)])], b"aaaa", "code"),
        "invalid_distance_code": ([Fixed([97, Match(259, 0, 31, 0)])], b"aaaa", "code"),
        "literal_code_without_symbol": ([Dynamic([Bits(1, 1)], **dict(lit_lens=_lens({256: 1}, 257), dist_lens=[0]), eob=False)], b"", "code"),
        "distance_code_without_symbol": ([Dynamic(tm + [257, Bits(1, 1)], dist_lens=_lens({6: 1}, 7), lit_lens=lit_m)], tm_text, "code"),
        "match_with_empty_distance_tree": ([Dynamic(t[:9] + [257, Bits(0, 1)], dist_lens=[0], lit_lens=lit_m)], tm_text, "code"),
        "distance_before_start": ([Fixed([97, (3, 2)])], b"aaaa", "distance"),
    }
    return {k: (deflate(v) if isinstance(v, list) else v, x, e) for k, (v, x, e) in m.items()}


# ----------------------------------------------------------------------------- seeded random streams for the differential test against zlib
DIFF_SEEDS = (1, 2, 3)
DIFF_BASES = 300                                                        # valid streams per seed, each followed by two mutations of it


def _random_blocks(rng, fq):
    """1..4 random blocks of at most BGZF_MAX_TEXT bytes of text in all: stored, fixed or dynamic (random code lengths, limits, run-length
    coding and header sizes), literals from FASTQ text or an adversarial alphabet."""
    alphabets = [range(256), b"A", b"AC", b"ACGT\n", bytes([0, 255]), bytes(range(250, 256)) + b"A" * 40]
    budget = [0, 2000, 12_000, BGZF_MAX_TEXT][rng.choice([1, 1, 1, 2, 2, 3])]
    blocks, pos = [], 0
    for _ in range(rng.randint(1, 4)):
        size = rng.randint(0, max(0, (budget - pos) // 2))
        kind = rng.choice(["stored", "fixed", "dynamic", "dynamic", "dynamic"])
        if rng.random() < 0.5:
            lit = _lit_seq(fq, rng.randrange(len(fq) - 1))
        else:
            lit = _lit_from(rng, rng.choice(alphabets))
        if kind == "stored":
            blocks.append(Stored(bytes(lit() for _ in range(size))))
        else:
            lsyms = range(257, 257 + rng.randint(1, 29))
            dsyms = range(rng.randint(0, 29), 30) if rng.random() < 0.5 else range(rng.randint(1, 30))
            toks = random_tokens(rng, size, lit, pos0=pos, match_rate=rng.choice([0, 0.1, 0.3, 0.6]), lsyms=lsyms, dsyms=dsyms)
            if kind == "fixed":
                blocks.append(Fixed(toks))
            else:
                lf, df = [0] * 286, [0] * 30                           # the tokens' counts, plus noise on symbols they do not use
                for tk in toks + [256]:
                    if isinstance(tk, int):
                        lf[tk] += 1
                    else:
                        lf[tk.lsym] += 1
                        df[tk.dsym] += 1
                for _ in range(rng.choice([0, 3, 30, 300])):
                    lf[rng.randrange(286)] += rng.randint(1, 3)
                for _ in range(rng.choice([0, 0, 2, 20])):
                    df[rng.randrange(30)] += 1
                if rng.random() < 0.3:                                   # skew: some codes reach the length limit
                    for s in range(286):
                        lf[s] = lf[s] * (1 << rng.randrange(12)) if lf[s] else 0
                lim = rng.choice([9, 10, 11, 12, 15])
                blocks.append(Dynamic(toks, huffman_lengths(lf, lim), huffman_lengths(df, rng.choice([5, 8, 9, 15])),
                                      hlit=rng.choice([None, None, 286]), hdist=rng.choice([None, None, 30]),
                                      hclen=rng.choice([None, None, 19]), rle=rng.choice(["plain", "runs", "cross"])))
        pos += size
    return blocks


def _mutate(rng, data, layout):
    """A mutation of a valid stream: 1..3 bit flips, mostly in block headers and code-length sections; a truncation; or appended bytes."""
    kind = rng.random()
    if kind < 0.6 and data:
        b = bytearray(data)
        for _ in range(rng.randint(1, 3)):
            if rng.random() < 0.8:
                start, first, end = rng.choice(layout)
                bit = rng.randrange(start, min(first + 16, end, len(b) * 8)) if min(first + 16, end, len(b) * 8) > start else 0
            else:
                bit = rng.randrange(len(b) * 8)
            b[bit // 8] ^= 1 << bit % 8
        return bytes(b)
    if kind < 0.8 and len(data) > 2:
        return data[:rng.randrange(2, len(data))]                       # a BGZF member holds at least 2 bytes of deflate data
    return data + bytes(rng.getrandbits(8) for _ in range(rng.randint(1, 4)))


def differential_streams(seed):
    """[(deflate data, text of the valid stream it was made from)]: DIFF_BASES valid streams from `seed`, each followed by two mutations.
    zlib's verdict on each decides what the kernel must do."""
    import random
    rng = random.Random(seed)
    fq = _fq_source(9000 + seed)
    out = []
    for i in range(DIFF_BASES):
        while True:
            blocks = _random_blocks(rng, fq)
            data = deflate(blocks, seed=rng.getrandbits(32), layout=(layout := []))
            if len(data) <= BGZF_MAX_DATA - 4:                             # room for 4 appended bytes
                break
        text = blocks_text(blocks)
        out.append((data, text))
        for _ in range(2):
            out.append((_mutate(rng, data, layout), text))
    return out
