"""Homopolymer compression (`kmc -hc`) for the tests: the numpy model of the batch rule the GPU applies, a per-read transcription of the
reference's CSplitter::HomopolymerCompressSeq (kmc_core/splitter.cpp:424-435) to pin it to, seeded homopolymer-rich reads, and the cases
whose `kmc -hc -sr1` results tests/golden/make_hc_reference.py stores in tests/golden/hc_reference.json."""
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HC_GOLDEN = os.path.join(ROOT, "tests", "golden", "hc_reference.json")
HC_MAPS = os.path.join(ROOT, "tests", "golden", "hc_maps.npz")
# GetSeq cuts a read into parts of mem_part_pmm_reads = (2^16 + 1) * 8 symbols (kmc.h:419, splitter.cpp:143-147), each compressed on its
# own: byte identity with the reference holds for shorter records
PART_SYMBOLS = (2 ** 16 + 1) * 8

_CODE = np.full(256, 4, dtype=np.uint8)
for _i, _c in enumerate(b"ACGT"):
    _CODE[_c] = _CODE[_c + 32] = _i


# ------------------------------------------------------------------------------------------------ the model
def homopolymer_compress(batch):
    """The batch rule: byte i is dropped iff i > 0, it is one of ACGTacgt and byte i - 1 is the same base ignoring case (uint8 array)."""
    a = np.asarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)
    c = _CODE[a]
    drop = np.zeros(a.size, dtype=bool)
    drop[1:] = (c[1:] < 4) & (c[1:] == c[:-1])
    return a[~drop]


def padded(batch):
    """homopolymer_compress(batch) padded back to the batch's length with '\\n': what the GPU hands to the kernels after it."""
    a = np.asarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)
    c = homopolymer_compress(a)
    return np.concatenate([c, np.full(a.size - c.size, 10, dtype=np.uint8)])


def compress_read(read):
    """One read as the reference compresses it: GetSeq's codes (ACGT / acgt -> 0..3, any other byte -> -1), then every code equal to the
    last one kept is dropped, so runs of N (or of any other byte) collapse too.  Returns the kept bytes of the read."""
    out = bytearray()
    last = None
    for ch in bytes(read):
        code = int(_CODE[ch]) if _CODE[ch] < 4 else -1
        if last is None or code != last:
            out.append(ch)
            last = code
    return bytes(out)


# ------------------------------------------------------------------------------------------------ reads
_LETTERS = np.frombuffer(b"ACGT", dtype=np.uint8)


def _run(rng, base, n, mixed):
    r = bytes([base]) * n
    if mixed:
        low = rng.random(n) < 0.5
        r = bytes(ch + 32 if lo else ch for ch, lo in zip(r, low))
    return r


def _distinct_neighbours(rng, m):
    """m bases, no two neighbours equal: a sequence that compresses to itself."""
    s = np.empty(m, dtype=np.uint8)
    prev = -1
    for i in range(m):
        b = int(rng.integers(0, 3))
        b = b + (b >= prev) if prev >= 0 else int(rng.integers(0, 4))
        s[i] = b
        prev = b
    return _LETTERS[s].tobytes()


def make_hc_reads(seed, profile, n_reads, read_len, k):
    """Seeded homopolymer-rich reads (list of bytes).  Read i is, by i % 8: a noisy genome sample with runs of 2..300 of one base put in;
    the same with mixed-case runs (aAAa); N / IUPAC runs and base runs next to them; one base repeated (some mixed case); a read that
    compresses to k - 1, k or k + 1 bases; a read that ends in a run whose base the next read starts with.  The only profile is "hp";
    the lengths of the genome samples vary from read_len / 3 to read_len."""
    rng = np.random.default_rng(seed)
    genome = _LETTERS[rng.integers(0, 4, 100_000 + read_len)]
    reads = []
    carry = None                                                       # the base the next read starts with (kind 5)
    for i in range(n_reads):
        kind = i % 8
        assert profile == "hp", profile
        n = int(rng.integers(max(1, read_len // 3), read_len + 1))
        if kind == 3:
            r = _run(rng, int(_LETTERS[rng.integers(0, 4)]), int(rng.integers(1, 301)), i % 16 == 3)
        elif kind == 4:
            m = k - 1 + (i // 8) % 3
            r = b"".join(_run(rng, ch, int(rng.integers(1, 6)), bool(rng.integers(0, 2))) for ch in _distinct_neighbours(rng, max(m, 1)))
        else:
            p = int(rng.integers(0, genome.size - n))
            s = genome[p:p + n].copy()
            s[rng.random(n) < 0.01] = _LETTERS[rng.integers(0, 4)]
            r = s.tobytes()
            pieces, pos = [], 0
            for _ in range(int(rng.integers(2, 9))):
                at = int(rng.integers(pos, max(pos + 1, len(r))))
                pieces.append(r[pos:at])
                ln = int(rng.integers(2, 13)) if rng.random() < 0.8 else int(rng.integers(13, 301))
                base = r[at] if at < len(r) else int(_LETTERS[rng.integers(0, 4)])
                if kind == 2 and rng.random() < 0.5:
                    pieces.append(_run(rng, base, ln // 2 + 1, False) + rng.choice(np.frombuffer(b"NNNRYn", dtype=np.uint8), int(rng.integers(1, 20))).tobytes()
                                  + _run(rng, base, ln // 2 + 1, False))
                else:
                    pieces.append(_run(rng, base, ln, kind == 1))
                pos = at
            pieces.append(r[pos:])
            r = b"".join(pieces)
        if carry is not None:
            r = _run(rng, carry, int(rng.integers(1, 8)), False) + r
            carry = None
        if kind == 5:
            carry = int(_LETTERS[rng.integers(0, 4)])
            r = r + _run(rng, carry, int(rng.integers(2, 30)), False)
        reads.append(r)
    return reads


# ------------------------------------------------------------------------------------------------ stored reference cases
# name: (seed, read profile, n_reads, read_len, k, kmc options); the reference runs with -hc -sr1 added.  The bin-path cases choose their
# map from the reads (no map given): -n64 unless the case keeps the default -n.  -fa / -fm: FASTA, one line / 60 bases a line (LF).
HC_CASES = {
    "k17_p7": (301, "hp", 1500, 200, 17, ("-p7", "-ci1", "-n64")),
    "k28_p9": (302, "hp", 1500, 200, 28, ("-p9", "-ci1", "-n64")),
    "k31_p9": (303, "hp", 1500, 200, 31, ("-p9", "-ci2", "-n64")),
    "k31_p11_b": (304, "hp", 1500, 200, 31, ("-p11", "-ci1", "-b", "-n64")),
    "k32_p9": (305, "hp", 1500, 200, 32, ("-p9", "-ci1", "-n64")),
    "k55_p11": (306, "hp", 1200, 250, 55, ("-p11", "-ci1", "-n64")),
    "k64_p7_b": (307, "hp", 1200, 250, 64, ("-p7", "-ci1", "-b", "-n64")),
    "k128_p9": (308, "hp", 800, 400, 128, ("-p9", "-ci1", "-n64")),
    "k31_p9_mix": (309, "hp", 1500, 200, 31, ("-p9", "-ci2", "-cx40", "-cs20", "-n64")),
    "k31_p9_n512": (310, "hp", 1500, 200, 31, ("-p9", "-ci1")),
    "k31_p9_opt": (311, "hp", 1500, 200, 31, ("-p9", "-ci1", "-n64", "--opt-out-size")),
    "k31_p9_fa": (312, "hp", 1200, 200, 31, ("-p9", "-ci1", "-n64", "-fa")),
    "k31_p9_fm": (313, "hp", 1200, 300, 31, ("-p9", "-ci1", "-n64", "-fm")),
    # small k: KMC's small-k path (no bins); -m4 leaves room for the 4^13 counters, or the reference falls back to bins
    "k1_small": (321, "hp", 1000, 150, 1, ("-ci1", "-m4")),
    "k5_small": (322, "hp", 1000, 150, 5, ("-ci1", "-m4")),
    "k11_small_b": (323, "hp", 1000, 150, 11, ("-ci1", "-b", "-m4")),
    "k13_small": (324, "hp", 1000, 150, 13, ("-ci2", "-m4")),
    # `kmc -e -hc`: the estimate of the uncompressed reads
    "k31_e": (331, "hp", 1500, 200, 31, ("-e",)),
}


def case_reads(name):
    seed, profile, n_reads, read_len, k, _ = HC_CASES[name]
    return make_hc_reads(seed, profile, n_reads, read_len, k)


def case_format(name):
    opts = HC_CASES[name][5]
    return "-fm" if "-fm" in opts else "-fa" if "-fa" in opts else "-fq"


def write_case_input(name, path):
    """The case's reads as the file the reference counts: FASTQ, or FASTA with one line (-fa) or 60 bases (-fm) a line."""
    reads = case_reads(name)
    fmt = case_format(name)
    with open(path, "wb") as f:
        for i, r in enumerate(reads):
            if fmt == "-fq":
                f.write(b"@r%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)))
            else:
                line = len(r) + 1 if fmt == "-fa" else 60
                f.write(b">r%d\n" % i + b"\n".join(r[j:j + line] for j in range(0, max(len(r), 1), line)) + b"\n")


def case_options(name):
    """The case's options without the input format: what follows -k in the reference's command line."""
    return [o for o in HC_CASES[name][5] if o not in ("-fa", "-fm")]


def option(name, flag, default):
    for o in HC_CASES[name][5]:
        if o.startswith(flag) and o[len(flag):].isdigit():
            return int(o[len(flag):])
    return default


def golden():
    return json.load(open(HC_GOLDEN))


def load_map(name):
    return np.load(HC_MAPS)[name].astype(np.uint32)
