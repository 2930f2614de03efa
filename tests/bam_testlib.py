"""Seeded BAM files for the BAM input tests: records packed with struct as the SAM/BAM specification lays them out, BGZF members through
gzip_testlib's writer, in the member layouts real writers use (htslib ends members on records, htsjdk does not, records over 64 KiB
straddle members by necessity), and adversarial records whose names, qualities and tags hold well-formed fixed fields at many offsets.
tests/golden/bam_reference.json holds what the reference CLI (`kmc -fbam`) makes of BAM_CASES."""
import os
import struct

import numpy as np

from gzip_testlib import BGZF_EOF, bgzf_member

BAM_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bam_reference.json")
CODES = b"=ACMGRSVTWYHKDBN"
_CODE = {c: i for i, c in enumerate(CODES)}
BGZF_FIXED_PIECE = 65280                                                # what htslib and htsjdk put in one member, at most
LAYOUTS = ("aligned", "fixed", "random")
_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def encode_seq(seq):
    """SEQ letters (=ACMGRSVTWYHKDBN) -> the 4-bit codes, two to a byte, high nibble first."""
    c = [_CODE[x] for x in seq] + ([0] if len(seq) % 2 else [])
    return bytes((c[i] << 4) | c[i + 1] for i in range(0, len(c), 2))


def record(name, flag, seq, n_cigar=1, qual=None, tags=b"", ref_id=0, pos=0, mapq=60):
    """One BAM record: block_size, the 32 bytes of fixed fields, the NUL-terminated name, CIGAR, SEQ, QUAL and tags."""
    cigar = b"".join(struct.pack("<I", (max(1, len(seq)) << 4) if i == 0 else (1 << 4) | 2) for i in range(n_cigar))
    qual = b"\xff" * len(seq) if qual is None else qual
    assert len(qual) == len(seq)
    body = struct.pack("<iiBBHHHiiii", ref_id, pos, len(name) + 1, mapq, 4680, n_cigar, flag, len(seq), -1, -1, 0) + name + b"\0" + cigar \
        + encode_seq(seq) + qual + tags
    return struct.pack("<i", len(body)) + body


def header(text=b"", refs=()):
    """BAM\\1, l_text, the text, n_ref and each reference's l_name, NUL-terminated name and l_ref."""
    out = [b"BAM\1", struct.pack("<i", len(text)), text, struct.pack("<i", len(refs))]
    for name, length in refs:
        out += [struct.pack("<i", len(name) + 1), name + b"\0", struct.pack("<i", length)]
    return b"".join(out)


def big_header(n_refs=5000):
    """A header of many @SQ lines and references: it spans several members and reader pieces."""
    refs = [(b"chr%d_with_a_long_scaffold_name" % i, 1000 + i) for i in range(n_refs)]
    text = b"@HD\tVN:1.6\tSO:unsorted\n" + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % r for r in refs)
    return header(text, refs)


def b_array_tag(rng, n):
    return b"XBBC" + struct.pack("<i", n) + rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def flag_of(rng):
    """A FLAG mix: unmapped, reverse, secondary, supplementary, duplicate and QC-fail records."""
    f = 0
    for bit, p in ((0x10, 0.5), (0x100, 0.06), (0x800, 0.06), (0x4, 0.1), (0x400, 0.08), (0x200, 0.05), (0x1, 0.3), (0x40, 0.15)):
        if rng.random() < p:
            f |= bit
    return f


def reads_to_records(rng, reads, names=True):
    """The records of reads: FLAG 0x10 stores the reverse complement (as an aligner does), names, CIGAR ops and tags of varied size."""
    out = []
    for i, r in enumerate(reads):
        flag = flag_of(rng)
        seq = r.translate(_COMP)[::-1] if flag & 0x10 else r
        name = (b"read%d" % i) if names and rng.random() < 0.9 else (b"x" * 254)
        tags = b_array_tag(rng, int(rng.integers(0, 40))) if rng.random() < 0.5 else b"NMC\x01"
        out.append(record(name, flag, seq, n_cigar=int(rng.integers(1, 4)) if rng.random() < 0.95 else 300, tags=tags,
                          qual=bytes(rng.integers(0, 42, len(seq), dtype=np.uint8))))
    return out


def odd_records(seed, n=300):
    """Records of every kind the parser must decode: '=', IUPAC codes, odd and zero l_seq, 254-byte names, many CIGAR ops, B arrays."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = int(rng.choice([0, 1, 2, 3, 31, 150, 151, int(rng.integers(1, 600))]))
        alphabet = CODES if rng.random() < 0.3 else b"ACGT"
        seq = bytes(rng.choice(np.frombuffer(alphabet, dtype=np.uint8), L)) if L else b""
        name = b"n" * int(rng.choice([1, 10, 254]))
        out.append(record(name, flag_of(rng), seq, n_cigar=int(rng.choice([0, 1, 7, 500])), tags=b_array_tag(rng, int(rng.integers(0, 300)))))
    return out


def fake_fields(rng, l_seq=4):
    """A well-formed little record (name, NUL, SEQ) to hide inside the bytes of another one."""
    return record(b"f", 0, b"ACGT"[:l_seq], n_cigar=0, qual=b"\x10" * l_seq)


def adversarial_records(seed, n=40, length=3000):
    """Long records whose QUAL and B-array tags are tiled with well-formed little records at every few offsets: most positions in a
    tile that look like a record start are not one, so the tile guesses are wrong and the parser's resolve walks the tiles again."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        seq = bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), length))
        fake = fake_fields(rng)
        step = int(rng.integers(0, 7))
        qual = ((b"\x00" * step + fake) * (length // (len(fake) + step) + 1))[:length]
        tag = b"XFBC" + struct.pack("<i", 2 * len(fake)) + fake + fake
        out.append(record(b"adv%d" % i, flag_of(rng) & ~0x900, seq, qual=qual, tags=tag))
    return out


def long_records(seed, n, length):
    """Records of `length` random bases (HiFi-like reads from 15 kb; from 64 KiB on a record straddles BGZF members)."""
    rng = np.random.default_rng(seed)
    return [record(b"m64011/%d/ccs" % i, flag_of(rng), bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), length)),
                   qual=bytes(rng.integers(0, 94, length, dtype=np.uint8))) for i in range(n)]


def bgzf_text(text, layout, bounds=(), seed=0):
    """Decompressed BAM -> BGZF members + the EOF member.  aligned: members end on the given record bounds (htslib), records over a
    member's room split; fixed: 65,280-byte pieces whatever the records (htsjdk); random: seeded sizes of 0..65,280."""
    if layout == "aligned":
        pieces, start, last = [], 0, 0
        for b in list(bounds) + [len(text)]:
            if b - start > BGZF_FIXED_PIECE and last > start:
                pieces.append((start, last))
                start = last
            while b - start > BGZF_FIXED_PIECE:
                pieces.append((start, start + BGZF_FIXED_PIECE))
                start += BGZF_FIXED_PIECE
            last = b
        if len(text) > start:
            pieces.append((start, len(text)))
    elif layout == "fixed":
        pieces = [(i, min(i + BGZF_FIXED_PIECE, len(text))) for i in range(0, len(text), BGZF_FIXED_PIECE)]
    else:
        rng = np.random.default_rng(seed)
        pieces, i = [], 0
        while i < len(text):
            n = int(rng.integers(0, BGZF_FIXED_PIECE + 1))
            pieces.append((i, min(i + n, len(text))))
            i += n
    return b"".join(bgzf_member(text[a:b], level=1) for a, b in pieces) + BGZF_EOF


def bam_file(hdr, records, layout="aligned", seed=0):
    """(compressed file bytes, decompressed text) of a BAM file of these records."""
    text = hdr + b"".join(records)
    bounds, pos = [len(hdr)], len(hdr)
    for r in records:
        pos += len(r)
        bounds.append(pos)
    return bgzf_text(text, layout, bounds, seed), text


def case_reads(seed, n_reads=6000, read_len=150):
    from stage1_testlib import make_reads
    return make_reads(seed, "short", n_reads=n_reads, read_len=read_len)


# name -> (k, reference options besides -k / -fbam / -sr1, count_reads keywords)
BAM_CASES = {
    "k11_small": (11, [], {"small_k": True}),
    "k11_small_b": (11, ["-b"], {"small_k": True, "both_strands": False}),
    "k25": (25, [], {}),
    "k31": (31, [], {}),
    "k31_b": (31, ["-b"], {"both_strands": False}),
    "k31_hc": (31, ["-hc"], {"homopolymer_compressed": True}),
    "k31_b_hc": (31, ["-b", "-hc"], {"both_strands": False, "homopolymer_compressed": True}),
    "k31_ci1_cs7": (31, ["-ci1", "-cs7"], {"cutoff_min": 1, "counter_max": 7}),
    "k55": (55, [], {}),
    "k55_b": (55, ["-b"], {"both_strands": False}),
    "k128": (128, [], {}),
    "k31_e": (31, ["-e"], {}),
}


def case_bam(layout="aligned"):
    """(compressed, decompressed) of the golden cases' input: reads of the 'short' profile with a FLAG mix, a multi-member header."""
    rng = np.random.default_rng(2041)
    return bam_file(big_header(400), reads_to_records(rng, case_reads(2040)), layout, seed=7)


def bgzf_member_extra(text, extra=b"XY\x02\x00ab"):
    """A BGZF member whose gzip header holds another extra subfield before BC, as the SAM specification allows."""
    import zlib
    from gzip_testlib import deflate_raw
    data = deflate_raw(text, level=1)
    xlen = len(extra) + 6
    head = struct.pack("<BBBBIBBH", 31, 139, 8, 4, 0, 0, 255, xlen) + extra + struct.pack("<BBHH", 66, 67, 2, 12 + xlen + len(data) + 8 - 1)
    return head + data + struct.pack("<II", zlib.crc32(text), len(text) & 0xFFFFFFFF)
