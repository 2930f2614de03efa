"""CPU: a numpy model of the GPU reads-text parser's chunk contract (kmcb200_fastx_parse / kmc_b200.FastxParser), written from
kmc_b200.reads.sequences_to_batch and _record_end, and checked against them here.  tests/test_gpu_fastx.py compares the GPU with this
model and with sequences_to_batch.

    parse_chunk(raw, fmt, is_final, limit) -> (batch, consumed)

  * FASTQ: line 1 of every 4 (lines counted from the chunk's start) is kept with its '\\n'; records end after every 4th line.
  * FASTA: a header line becomes its '\\n', other lines are kept without theirs, blank lines vanish; records end where a header line starts
    after a '\\n' (never at an unterminated last line of a final chunk: _record_end's rule).
  * A final chunk is parsed to its end (as if it ended in '\\n'); a non-final one to its last record end, and one without a record end is an
    error.  With limit < len(raw): up to the first record end at or past limit when the chunk has one.
"""
import numpy as np
import pytest

from kmc_b200 import ERR_INVALID, FASTA, FASTQ, KmcB200Error
from kmc_b200.reads import _record_end, sequences_to_batch

NL, GT = 10, ord(">")
TOO_LONG = "a record is longer than the chunk"


# ----------------------------------------------------------------------------- the model
def to_batch(a, fmt):
    """sequences_to_batch with the format given instead of read from the first non-empty line."""
    a = np.asarray(a, dtype=np.uint8)
    if a.size == 0:
        return np.zeros(0, dtype=np.uint8)
    if a[-1] != NL:
        a = np.append(a, np.uint8(NL))
    ends = np.flatnonzero(a == NL)
    starts = np.concatenate([[0], ends[:-1] + 1])
    delta = np.zeros(a.size + 1, dtype=np.int64)
    if fmt == FASTQ:
        seq = np.arange(1, ends.size, 4)
        delta[starts[seq]] += 1
        delta[ends[seq] + 1] -= 1
        keep = np.cumsum(delta[:-1]) > 0
    else:
        hdr = np.flatnonzero(a[starts] == GT)
        delta[starts[hdr]] += 1
        delta[ends[hdr]] -= 1
        keep = np.cumsum(delta[:-1]) == 0
        keep[ends] = False
        keep[ends[hdr]] = True
    return a[keep]


def record_ends(a, fmt, is_final, reference_rule=True):
    """Record ends (exclusive) of a chunk.  reference_rule: drop a FASTA header start that begins an unterminated last line of a final
    chunk, as _record_end does; without it, every record start after the first is counted (what `records` reports)."""
    nl = np.flatnonzero(a == NL)
    if fmt == FASTQ:
        ends = nl[3::4] + 1
    else:
        q = nl[nl + 1 < a.size]
        ends = q[a[q + 1] == GT] + 1
        if reference_rule and is_final and a.size and a[-1] != NL and ends.size and ends[-1] == nl[-1] + 1:
            ends = ends[:-1]
    if is_final and a.size and (ends.size == 0 or ends[-1] != a.size):
        ends = np.append(ends, a.size)
    return ends


def cut_of(a, fmt, is_final, limit=None):
    ends = record_ends(a, fmt, is_final)
    if limit is not None and limit < a.size:
        past = ends[ends >= limit]
        if past.size:
            return int(past[0])
    if is_final:
        return int(a.size)
    if ends.size == 0:
        raise KmcB200Error(ERR_INVALID, TOO_LONG)
    return int(ends[-1])


def parse_chunk(raw, fmt, is_final, limit=None):
    """-> (batch uint8, consumed)"""
    a = np.frombuffer(bytes(raw), dtype=np.uint8)
    c = cut_of(a, fmt, is_final, limit)
    return to_batch(a[:c], fmt), c


def records_of(raw, fmt, consumed):
    """Records in raw[:consumed] (the parser's result word [2])."""
    a = np.frombuffer(bytes(raw), dtype=np.uint8)
    if consumed == 0:
        return 0
    ends = record_ends(a, fmt, False, reference_rule=False)
    return 1 + int((ends < consumed).sum())


def parse_in_chunks(data, fmt, chunk_ends, parse=parse_chunk):
    """Chunks that end at the given positions (the last one at len(data) is final), each starting where the previous one's parse stopped;
    a chunk without a record end is read on to the next position, as a caller with a larger buffer would.  -> (concatenated batches,
    chunk starts)."""
    out, pos, starts = [], 0, []
    for end in sorted(set(chunk_ends) | {len(data)}):
        if end <= pos:
            continue
        try:
            seq, c = parse(data[pos:end], fmt, end == len(data))
        except KmcB200Error as e:
            if TOO_LONG not in str(e) or end == len(data):
                raise
            continue
        starts.append(pos)
        out.append(np.asarray(seq, dtype=np.uint8))
        pos += c
    return (np.concatenate(out) if out else np.zeros(0, np.uint8)), starts


# ----------------------------------------------------------------------------- seeded inputs (the GPU tests use the same)
PHRED = np.arange(33, 75, dtype=np.uint8)                             # '!' .. 'J': holds '@', '+', '>', 'A', 'C', 'G'
BASES = np.frombuffer(b"ACGTACGTACGTNacgtRY", dtype=np.uint8)


def fastq_text(seed, n, max_len=300, crlf=False, final_newline=True, empty=True):
    """FASTQ with quality strings over the whole Phred+33 range '!'..'J', some empty sequences and headers, optional CRLF."""
    rng = np.random.default_rng(seed)
    eol = b"\r\n" if crlf else b"\n"
    recs = []
    for i in range(n):
        ln = int(rng.integers(0, max_len + 1)) if (empty and rng.random() < 0.05) else int(rng.integers(1, max_len + 1))
        seq = BASES[rng.integers(0, BASES.size, ln)].tobytes()
        qual = PHRED[rng.integers(0, PHRED.size, ln)].tobytes()
        name = b"" if (empty and rng.random() < 0.05) else b"r%d %s" % (i, PHRED[rng.integers(0, PHRED.size, 8)].tobytes())
        plus = b"+" + (name if rng.random() < 0.2 else b"")
        recs.append(b"@" + name + eol + seq + eol + plus + eol + qual + eol)
    text = b"".join(recs)
    return text if final_newline else text[:-len(eol)]


def fasta_text(seed, n, max_len=400, crlf=False, final_newline=True):
    """FASTA: 60-column lines, one line per record, blank lines, headers that are just '>', empty records, optional CRLF."""
    rng = np.random.default_rng(seed)
    eol = b"\r\n" if crlf else b"\n"
    out = []
    for i in range(n):
        ln = int(rng.integers(0, max_len + 1))
        seq = BASES[rng.integers(0, BASES.size, ln)].tobytes()
        width = [60, 80, max(ln, 1)][int(rng.integers(0, 3))]
        hdr = b">" if rng.random() < 0.1 else b">s%d desc ACGT>@+" % i
        lines = [seq[j:j + width] for j in range(0, ln, width)]
        if rng.random() < 0.15:
            lines.insert(int(rng.integers(0, len(lines) + 1)), b"")       # a blank line
        out.append(eol.join([hdr] + lines) + eol)
    text = b"".join(out)
    return text if final_newline else text[:-len(eol)]


def profile_text(seed, profile, fmt, n=300, read_len=150):
    """stage1_testlib.make_reads profiles ('n_dense', 'low_complexity', ...) as FASTQ or FASTA text."""
    from stage1_testlib import make_reads
    reads = make_reads(seed, profile, n_reads=n, read_len=read_len)
    if fmt == FASTQ:
        return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)) for i, r in enumerate(reads))
    return b"".join(b">r%d\n" % i + b"\n".join(r[j:j + 60] for j in range(0, max(len(r), 1), 60)) + b"\n" for i, r in enumerate(reads))


def corpus():
    """(name, text, fmt) of every seeded input shape."""
    return [
        ("fastq_phred", fastq_text(1, 400), FASTQ),
        ("fastq_crlf", fastq_text(2, 300, crlf=True), FASTQ),
        ("fastq_no_final_newline", fastq_text(3, 200, final_newline=False), FASTQ),
        ("fastq_crlf_no_final_newline", fastq_text(4, 100, crlf=True, final_newline=False), FASTQ),
        ("fasta", fasta_text(5, 300), FASTA),
        ("fasta_crlf", fasta_text(6, 200, crlf=True), FASTA),
        ("fasta_no_final_newline", fasta_text(7, 150, final_newline=False), FASTA),
        ("fasta_header_last", fasta_text(8, 50) + b">last header", FASTA),
        ("fastq_n_dense", profile_text(9, "n_dense", FASTQ), FASTQ),
        ("fasta_low_complexity", profile_text(10, "low_complexity", FASTA, n=20, read_len=3000), FASTA),
    ]


def special_cuts(data, fmt):
    """Chunk ends at the awkward places: 1 byte past a record end, exactly one record, between '\\r' and '\\n'."""
    a = np.frombuffer(data, dtype=np.uint8)
    ends = record_ends(a, fmt, False)
    cuts = []
    if ends.size > 3:
        cuts += [int(ends[0]) + 1, int(ends[2])]                       # the second chunk holds exactly records 1..2 -> then one record
        cuts += [int(ends[3])]
    cr = np.flatnonzero((a[:-1] == 13) & (a[1:] == NL))
    if cr.size:
        cuts.append(int(cr[cr.size // 2]) + 1)                          # between '\r' and '\n'
    return sorted(c for c in set(cuts) if 0 < c < a.size)


def random_cuts(rng, n, lo, hi):
    cuts, pos = [], 0
    while True:
        pos += int(rng.integers(lo, hi))
        if pos >= n:
            return cuts
        cuts.append(pos)


def longest_record(data, fmt):
    a = np.frombuffer(data, dtype=np.uint8)
    ends = np.concatenate([[0], record_ends(a, fmt, True)])
    return int(np.diff(ends).max())


# ----------------------------------------------------------------------------- the model against sequences_to_batch / _record_end
CORPUS = corpus()


@pytest.mark.parametrize("name,data,fmt", CORPUS, ids=[c[0] for c in CORPUS])
def test_model_whole_file_is_sequences_to_batch(name, data, fmt):
    seq, c = parse_chunk(data, fmt, True)
    assert c == len(data)
    assert seq.tobytes() == sequences_to_batch(data).tobytes()


@pytest.mark.parametrize("name,data,fmt", CORPUS, ids=[c[0] for c in CORPUS])
def test_chunks_concatenate_to_sequences_to_batch(name, data, fmt):
    want = sequences_to_batch(data).tobytes()
    got, starts = parse_in_chunks(data, fmt, special_cuts(data, fmt))
    assert got.tobytes() == want
    assert len(starts) > 1
    rng = np.random.default_rng(len(data))
    longest = longest_record(data, fmt)
    for trial in range(20):
        lo = longest + 1 if trial % 2 else 1
        cuts = random_cuts(rng, len(data), lo, lo + int(rng.integers(1, 3 * longest + 2)))
        got, starts = parse_in_chunks(data, fmt, cuts)
        assert got.tobytes() == want, (trial, cuts[:5])


def test_special_cuts_hit_the_awkward_places():
    data = fastq_text(2, 300, crlf=True)
    a = np.frombuffer(data, dtype=np.uint8)
    cuts = special_cuts(data, FASTQ)
    ends = record_ends(a, FASTQ, False)
    assert int(ends[0]) + 1 in cuts and int(ends[2]) in cuts and int(ends[3]) in cuts
    assert any(a[c - 1] == 13 and a[c] == NL for c in cuts)
    _, starts = parse_in_chunks(data, FASTQ, cuts)
    assert {0, int(ends[0]), int(ends[2]), int(ends[3])} <= set(starts)  # chunks start on records; [ends[2], ends[3]) is one record


@pytest.mark.parametrize("name,data,fmt", CORPUS, ids=[c[0] for c in CORPUS])
def test_limit_is_the_sample_cut(name, data, fmt):
    rng = np.random.default_rng(7 + len(data))
    limits = [1, 2, len(data) - 1, len(data)] + [int(x) for x in rng.integers(1, len(data), 40)]
    for limit in limits:
        seq, c = parse_chunk(data, fmt, True, limit)
        cut = _record_end(data, limit - 1)
        assert c == cut, limit
        assert seq.tobytes() == sequences_to_batch(data[:cut]).tobytes(), limit


def test_limit_in_a_non_final_chunk_without_a_record_end_past_it():
    data = fastq_text(11, 20)
    a = np.frombuffer(data, dtype=np.uint8)
    ends = record_ends(a, FASTQ, False)
    chunk = data[:int(ends[5]) + 10]                                   # ends 10 bytes into record 6
    seq, c = parse_chunk(chunk, FASTQ, False, limit=int(ends[5]) + 3)
    assert c == int(ends[5])                                            # parsed to its last record end: consumed < limit, go on
    seq, c = parse_chunk(chunk, FASTQ, False, limit=int(ends[2]) - 1)
    assert c == int(ends[2])


def test_a_chunk_without_a_record_end_is_an_error():
    for data, fmt in ((fastq_text(12, 3), FASTQ), (fasta_text(13, 3), FASTA)):
        a = np.frombuffer(data, dtype=np.uint8)
        first = int(record_ends(a, fmt, False)[0])
        with pytest.raises(KmcB200Error) as ei:
            parse_chunk(data[:first - 1], fmt, False)
        assert ei.value.code == ERR_INVALID and TOO_LONG in str(ei.value)
        seq, c = parse_chunk(data[:first - 1], fmt, True)                # the same bytes as a final chunk are fine
        assert c == first - 1
    with pytest.raises(KmcB200Error):
        parse_chunk(b">only one record\nACGT\nACGT\n", FASTA, False)     # FASTA: a record ends only where the next header starts


def test_output_never_exceeds_bytes_plus_one_and_records():
    for name, data, fmt in CORPUS:
        seq, c = parse_chunk(data, fmt, True)
        assert seq.size <= len(data) + 1
    assert parse_chunk(b"@r", FASTQ, True)[0].tobytes() == b""             # line 0 of 4 is the header: nothing kept
    assert parse_chunk(b"@r\nACGT", FASTQ, True)[0].tobytes() == b"ACGT\n"  # line 1, unterminated: kept with a '\n'
    assert parse_chunk(b"@r\nACGT\n+\nIIII", FASTQ, True)[0].tobytes() == b"ACGT\n"
    assert parse_chunk(b">h", FASTA, True)[0].tobytes() == b"\n"
    assert records_of(fastq_text(1, 37), FASTQ, len(fastq_text(1, 37))) == 37
    assert records_of(fasta_text(5, 41), FASTA, len(fasta_text(5, 41))) == 41
