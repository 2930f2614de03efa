"""CPU: the BAM host model (kmc_b200.reads.bam_to_batch and its helpers), which parse="host" runs and every GPU BAM test compares with.
The model's batches equal the ones tests/golden/bam_reference.json stores, which the reference CLI was checked to count exactly as its own
BAM reader does (tests/golden/make_bam_reference.py)."""
import hashlib
import json
import os
import struct

import numpy as np
import pytest

from bam_testlib import BAM_CASES, BAM_GOLDEN, LAYOUTS, adversarial_records, bam_file, bgzf_member_extra, big_header, case_bam, \
    encode_seq, header, long_records, odd_records, record
from gzip_testlib import BGZF_EOF, bgzf_member, write
from kmc_b200 import ERR_INVALID, KmcB200Error
from kmc_b200 import reads

GOLDEN = json.load(open(BAM_GOLDEN))
_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def naive_batch(records, original_strand):
    """A record-by-record restatement of CSplitter::GetSeq (splitter.cpp:326-418) on the writer's own records."""
    out = []
    for r in records:
        bs, = struct.unpack_from("<i", r, 0)
        l_name, n_cigar, flag, l_seq = r[12], *struct.unpack_from("<HHi", r, 16)
        if flag & 0x900:
            continue
        s = 36 + l_name + 4 * n_cigar
        seq = bytes(b"NACNGNNNTNNNNNNN"[(r[s + j // 2] >> (0 if j & 1 else 4)) & 15] for j in range(l_seq))
        if original_strand and flag & 0x10:
            seq = seq.translate(_COMP)[::-1]
        out.append(seq + b"\n")
    return b"".join(out)


def test_golden_batches_are_the_models():
    _, text = case_bam()
    for name, (k, opts, _) in BAM_CASES.items():
        g = GOLDEN[name]
        assert hashlib.md5(text).hexdigest() == g["bam_md5"], name
        batch = reads.bam_to_batch(text, original_strand="-b" in opts)
        assert hashlib.md5(batch.tobytes()).hexdigest() == g["batch_md5"], name


@pytest.mark.parametrize("kind", ["odd", "adversarial", "long"])
def test_model_equals_a_record_by_record_decode(kind):
    recs = {"odd": lambda: odd_records(5), "adversarial": lambda: adversarial_records(6, n=10),
            "long": lambda: long_records(7, 3, 70_000)}[kind]()
    text = header(b"@HD\tVN:1.6\n", [(b"chr1", 1000)]) + b"".join(recs)
    for orig in (False, True):
        assert reads.bam_to_batch(text, orig).tobytes() == naive_batch(recs, orig)


def test_codes_and_strands():
    recs = [record(b"a", 0, b"=ACMGRSVTWYHKDBN"), record(b"b", 0x10, b"ACGTN"), record(b"c", 0x100, b"AAAA"), record(b"d", 0x800, b"CC"),
            record(b"e", 0x4 | 0x400 | 0x200, b"G"), record(b"f", 0, b"")]
    text = header() + b"".join(recs)
    assert reads.bam_to_batch(text).tobytes() == b"NACNGNNNTNNNNNNN\nACGTN\nG\n\n"
    assert reads.bam_to_batch(text, True).tobytes() == b"NACNGNNNTNNNNNNN\nNACGT\nG\n\n"
    assert reads.bam_n_reads(reads.bam_records(text)) == 4
    assert encode_seq(b"ACG") == bytes([0x12, 0x40])


def test_header_is_skipped_across_any_pieces():
    hdr = big_header(300)
    text = hdr + b"".join(odd_records(8, 20))
    for piece in (1, 3, 4, 7, 1000, 65280):
        h = reads.BamHeader()
        at = None
        for i in range(0, len(text), piece):
            at = h.feed(text[i:i + piece])
            if at is not None:
                assert i + at == len(hdr)
                break
        assert at is not None
    assert len(reads.bam_records(header())) == 0
    with pytest.raises(KmcB200Error):
        reads.bam_records(hdr[:-3])


def _bad(text):
    with pytest.raises(KmcB200Error) as e:
        reads.bam_to_batch(text)
    assert e.value.code == ERR_INVALID


def test_malformed_records_are_errors():
    good = record(b"r", 0, b"ACGTACGT")
    h = header()
    _bad(b"BAM\2" + h[4:] + good)                                         # no magic
    _bad(h + struct.pack("<i", 31) + good[4:35])                            # block_size < 32
    over = bytearray(good)
    over[12] = 200                                                        # l_read_name past block_size
    _bad(h + bytes(over))
    neg = bytearray(good)
    neg[20:24] = struct.pack("<i", -1)                                    # negative l_seq
    _bad(h + bytes(neg))
    many = bytearray(good)
    many[16:18] = struct.pack("<H", 60000)                                # CIGAR ops past block_size
    _bad(h + bytes(many))
    _bad(h + good + good[:-1])                                            # truncated last record
    _bad(h + good + good[:3])                                             # a partial block_size


def test_files_must_be_bgzf_with_the_eof_member(tmp_path):
    raw, text = bam_file(header(), odd_records(9, 30), "fixed")
    assert reads.read_bam(write(str(tmp_path / "ok.bam"), raw)) == text
    for name, data in [("no_eof", raw[:-len(BGZF_EOF)]),
                       ("plain_gzip", __import__("gzip").compress(text) + BGZF_EOF),
                       ("not_bgzf_member", bgzf_member(text[:100]) + __import__("gzip").compress(text[100:]) + BGZF_EOF)]:
        with pytest.raises(KmcB200Error) as e:
            reads.read_bam(write(str(tmp_path / (name + ".bam")), data))
        assert e.value.code == ERR_INVALID, name


def test_members_with_other_extra_subfields_are_bgzf(tmp_path):
    """The host check walks the extra subfields as kmcb200_bgzf_scan does: a BC subfield after another one is still BGZF."""
    import kmc_b200
    _, text = bam_file(header(), odd_records(14, 30), "fixed")
    raw = bgzf_member_extra(text[:40000]) + bgzf_member_extra(text[40000:]) + BGZF_EOF
    assert reads.read_bam(write(str(tmp_path / "extra.bam"), raw)) == text
    used, n, members = kmc_b200.bgzf_scan(raw, len(text))
    assert used == len(raw) and n == len(text) and len(members) == 3
    bad = bytearray(raw)
    bad[18:20] = b"BD"                                                   # the first member's BC renamed: no BC subfield left
    with pytest.raises(KmcB200Error):
        reads.read_bam(write(str(tmp_path / "no_bc.bam"), bytes(bad)))


def test_detection_and_predicted_size(tmp_path):
    raw, _ = case_bam()
    bam = write(str(tmp_path / "reads.fq.gz"), raw)                       # the name does not matter
    fq = write(str(tmp_path / "reads.fq"), b"@r\nACGT\n+\nIIII\n")
    assert reads.is_bam(bam) and not reads.is_bam(fq)
    assert reads.predicted_size([bam]) == int(0.7 * len(raw))
    assert reads.predicted_size([bam, fq]) == int(0.7 * len(raw)) + os.path.getsize(fq)


def test_layouts_give_the_same_text():
    texts = {layout: case_bam(layout) for layout in LAYOUTS}
    assert len({t for _, t in texts.values()}) == 1
    assert len({r for r, _ in texts.values()}) == len(LAYOUTS)


def test_record_end_for_the_sample():
    recs = odd_records(10, 50)
    data = b"".join(recs)
    ends = np.cumsum([len(r) for r in recs])
    for at in (0, 1, int(ends[0]) - 1, int(ends[0]), int(ends[10]) + 5, len(data) - 1):
        assert reads.bam_record_end(data, at) == int(ends[np.searchsorted(ends, at, side="right")])
