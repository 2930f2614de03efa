"""GPU: BAM records parsed on the H100 (kmc_b200.FastxParser with BAM / BAM_ORIGINAL_STRAND, the _fastx entry points of every reads
handle, and count_reads / count_reads_small_k / estimate_histogram on BAM files).  Every parse is compared byte for byte with the host
model (kmc_b200.reads.bam_records_to_batch and the serial walk below), and the databases with tests/golden/bam_reference.json, which
holds the reference CLI's `kmc -fbam` files."""
import hashlib
import json
import struct

import numpy as np
import pytest

from bam_testlib import BAM_CASES, BAM_GOLDEN, adversarial_records, bam_file, big_header, case_bam, header, long_records, odd_records, \
    reads_to_records, record, case_reads
from gzip_testlib import write
from stage1_testlib import random_map

pytestmark = pytest.mark.gpu

TOO_LONG, TRUNCATED, MALFORMED = 1, 2, 3


def parser(fmt, max_chunk=1 << 22):
    import kmc_b200
    return kmc_b200.FastxParser(fmt, max_chunk_bytes=max_chunk)


def model_chunk(data, final, limit=None):
    """(batch, consumed, kept records) of one chunk of record bytes, or the error word: the walk the parser makes."""
    from kmc_b200.reads import bam_records_to_batch
    n, p, cut = len(data), 0, False
    while p < n:
        if n - p < 4:
            break
        bs, = struct.unpack_from("<i", data, p)
        if bs < 32:
            return MALFORMED
        if n - p - 4 < bs:
            break
        l_name, n_cigar, l_seq = data[p + 12], *struct.unpack_from("<H", data, p + 16), struct.unpack_from("<i", data, p + 20)[0]
        if l_seq < 0 or 32 + l_name + 4 * n_cigar + (l_seq + 1) // 2 + l_seq > bs:
            return MALFORMED
        p += 4 + bs
        if limit is not None and limit < n and p >= limit:
            cut = True
            break
    if p < n and final and not cut:
        return TRUNCATED
    if not final and p == 0:
        return TOO_LONG
    batch = bam_records_to_batch(bytes(data[:p]), False)
    return p, int(np.count_nonzero(batch == 10))


def records_of(seed):
    rng = np.random.default_rng(seed)
    return reads_to_records(rng, case_reads(seed, n_reads=800)) + odd_records(seed, 150) + adversarial_records(seed, 6) + \
        long_records(seed, 2, 40_000) + reads_to_records(rng, case_reads(seed + 1, n_reads=300))


CORPUS = {
    "mixed": lambda: b"".join(records_of(11)),
    "short": lambda: b"".join(reads_to_records(np.random.default_rng(3), case_reads(3, n_reads=3000))),
    "odd": lambda: b"".join(odd_records(4, 400)),
    "adversarial": lambda: b"".join(adversarial_records(5, 60)),
    "long": lambda: b"".join(long_records(6, 4, 150_000)),           # records spanning many tiles, tiles with no record start
    "one_record": lambda: record(b"only", 0x10, b"ACGTTGCA" * 3000),
    "empty_seqs": lambda: b"".join(record(b"e%d" % i, 0, b"") for i in range(2000)),
}


def _batch(data, orig):
    from kmc_b200.reads import bam_records_to_batch
    return bam_records_to_batch(data, orig).tobytes()


# ----------------------------------------------------------------------------- parse parity
@pytest.mark.parametrize("orig", [False, True])
@pytest.mark.parametrize("name", sorted(CORPUS))
def test_whole_chunk_equals_model(name, orig):
    import kmc_b200
    data = CORPUS[name]()
    p = parser(kmc_b200.BAM_ORIGINAL_STRAND if orig else kmc_b200.BAM)
    seq, c = p.parse(data, True)
    assert c == len(data)
    assert seq.tobytes() == _batch(data, orig)
    assert p.last_records() == model_chunk(data, True)[1]
    p.close()


def _cuts(data):
    """Chunk ends inside block_size, inside the fixed fields, inside names and at record ends."""
    from kmc_b200.reads import bam_walk
    starts = [r[0] for r in bam_walk(data)]
    cuts = set()
    for s in starts[::max(1, len(starts) // 40)]:
        for d in (0, 1, 2, 3, 4, 13, 20, 35, 36, 37):
            cuts.add(min(len(data), s + d))
    return sorted(c for c in cuts if c > 0)


def parse_in_chunks(p, data, ends, orig):
    """The chunks [start, end) for each end, carrying the unparsed rest as a reader does; returns the concatenated batch."""
    out, start = [], 0
    for end in list(ends) + [len(data)]:
        if end <= start and end != len(data):
            continue
        final = end == len(data)
        chunk = data[start:end]
        want = model_chunk(chunk, final)
        if isinstance(want, int):
            assert want == TOO_LONG
            with pytest.raises(Exception):
                p.parse(chunk, final)
            continue
        seq, c = p.parse(chunk, final)
        assert (c, p.last_records()) == want
        out.append(seq.tobytes())
        start += c
    assert start == len(data)
    return b"".join(out)


@pytest.mark.parametrize("orig", [False, True])
@pytest.mark.parametrize("name", ["mixed", "odd", "adversarial", "long"])
def test_chunked_parse_equals_model(name, orig):
    import kmc_b200
    data = CORPUS[name]()
    p = parser(kmc_b200.BAM_ORIGINAL_STRAND if orig else kmc_b200.BAM)
    want = _batch(data, orig)
    assert parse_in_chunks(p, data, _cuts(data), orig) == want
    rng = np.random.default_rng(len(data))
    for _ in range(4):
        ends = np.cumsum(rng.integers(1, 200_000, 60))
        assert parse_in_chunks(p, data, [int(e) for e in ends if e < len(data)], orig) == want
    p.close()


@pytest.mark.parametrize("name", ["mixed", "adversarial", "long", "short"])
def test_limits_and_final_flags_equal_model(name):
    import kmc_b200
    data = CORPUS[name]()
    p = parser(kmc_b200.BAM)
    rng = np.random.default_rng(7)
    for limit in [0, 1, 35, 36, 37] + [int(x) for x in rng.integers(1, len(data), 12)] + [len(data)]:
        for final in (False, True):
            for end in (len(data), max(1, int(rng.integers(limit + 1, len(data) + 1)) if limit < len(data) else len(data))):
                chunk = data[:end]
                fin = final and end == len(data)
                want = model_chunk(chunk, fin, limit)
                if isinstance(want, int):
                    with pytest.raises(kmc_b200.KmcB200Error):
                        p.parse(chunk, fin, limit)
                    continue
                seq, c = p.parse(chunk, fin, limit)
                assert (c, p.last_records()) == want, (limit, fin, end)
                assert seq.tobytes() == _batch(chunk[:c], False)
    p.close()


def test_device_twin_on_a_caller_stream_and_its_result_words():
    import torch
    import kmc_b200
    data = CORPUS["mixed"]()
    p = parser(kmc_b200.BAM_ORIGINAL_STRAND)
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    cut = len(data) - 100
    with torch.cuda.stream(s):
        d_raw = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
        d_seq = torch.full((len(data) + 1,), 7, dtype=torch.uint8, device=dev)
        d_res = torch.zeros(4, dtype=torch.int64, device=dev)
        p.dev_parse(d_raw.data_ptr(), cut, False, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), s.cuda_stream)
    s.synchronize()
    c, recs = model_chunk(data[:cut], False)
    want = _batch(data[:c], True)
    assert [int(x) for x in d_res.cpu()] == [c, len(want), recs, 0]
    assert d_seq[:len(want)].cpu().numpy().tobytes() == want
    with torch.cuda.stream(s):
        d_seq.fill_(7)
        p.dev_parse(d_raw.data_ptr(), cut, True, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), s.cuda_stream)
    s.synchronize()
    assert [int(x) for x in d_res.cpu()] == [0, 0, 0, TRUNCATED]
    assert int((d_seq != 7).sum()) == 0                                  # nothing written
    p.close()


# ----------------------------------------------------------------------------- errors
def malformed_cases():
    good = record(b"r", 0x10, b"ACGTACGTAC")
    over, neg, many = bytearray(good), bytearray(good), bytearray(good)
    over[12] = 200
    neg[20:24] = struct.pack("<i", -5)
    many[16:18] = struct.pack("<H", 60000)
    body = b"".join(odd_records(12, 80))
    return {
        "block_size_31": (body + struct.pack("<i", 31) + good[4:36] + good, True, MALFORMED),
        "block_size_negative": (body + struct.pack("<i", -1) + good[4:], True, MALFORMED),
        "name_past_block": (body + bytes(over) + good, True, MALFORMED),
        "negative_l_seq": (body + bytes(neg), False, MALFORMED),
        "cigar_past_block": (good + bytes(many) + body, True, MALFORMED),
        "truncated_last": (body + good[:-1], True, TRUNCATED),
        "partial_block_size": (body + good[:2], True, TRUNCATED),
        "too_long": (good[:-1], False, TOO_LONG),
    }


@pytest.mark.parametrize("name", sorted(malformed_cases()))
def test_malformed_input_is_an_error_and_the_handle_goes_on(name):
    import torch
    import kmc_b200
    data, final, code = malformed_cases()[name]
    assert model_chunk(data, final) == code
    p = parser(kmc_b200.BAM)
    with pytest.raises(kmc_b200.KmcB200Error) as e:
        p.parse(data, final)
    assert e.value.code == kmc_b200.ERR_INVALID
    dev = torch.device("cuda:0")
    d_raw = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
    d_seq = torch.full((len(data) + 1,), 7, dtype=torch.uint8, device=dev)
    d_res = torch.full((4,), 99, dtype=torch.int64, device=dev)
    p.dev_parse(d_raw.data_ptr(), len(data), final, None, d_seq.data_ptr(), d_seq.numel(), d_res.data_ptr(), None)
    torch.cuda.synchronize()
    assert [int(x) for x in d_res.cpu()] == [0, 0, 0, code]
    assert int((d_seq != 7).sum()) == 0
    good = CORPUS["mixed"]()
    seq, c = p.parse(good, True)
    assert c == len(good) and seq.tobytes() == _batch(good, False)
    p.close()


def test_create_rejects_other_formats():
    import kmc_b200
    for fmt in (0, 3, 6, 99):
        with pytest.raises(kmc_b200.KmcB200Error):
            parser(fmt)


# ----------------------------------------------------------------------------- launches
def test_launches_do_not_depend_on_the_size():
    import kmc_b200
    block = CORPUS["short"]()
    big = block * ((1 << 28) // len(block))
    p = parser(kmc_b200.BAM, max_chunk=1 << 28)
    one = record(b"a", 0, b"ACGT")
    n0 = p.kernel_launches()
    seq, c = p.parse(one, True)
    n1 = p.kernel_launches()
    assert seq.tobytes() == b"ACGT\n" and c == len(one)
    seq, c = p.parse(big, True)
    n2 = p.kernel_launches()
    assert n1 - n0 == n2 - n1 == 7
    assert c == len(big) and seq.size == len(_batch(block, False)) * (len(big) // len(block))
    assert seq[:len(_batch(block, False))].tobytes() == _batch(block, False)
    p.close()


# ----------------------------------------------------------------------------- consumers
def split_tuple(out, packs, frags):
    fr = np.array([[f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs] for f in frags], dtype=np.uint64)
    return out.tobytes(), packs.tobytes(), fr.tobytes()


@pytest.mark.parametrize("orig", [False, True])
def test_every_handle_takes_a_bam_parser(orig):
    import kmc_b200
    data = CORPUS["mixed"]()
    batch = np.frombuffer(_batch(data, orig), dtype=np.uint8)
    fmt = kmc_b200.BAM_ORIGINAL_STRAND if orig else kmc_b200.BAM
    p = parser(fmt)
    k, m, nb = 31, 9, 64
    sig_map = random_map(5, m, nb)
    cap = len(data) + 1
    sp, ref = (kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=cap) for _ in range(2))
    out, packs, frags, c, nseq = sp.split_fastx(p, data, True)
    assert c == len(data) and nseq == batch.size
    assert split_tuple(out, packs, frags) == split_tuple(*ref.split_raw(batch))
    st, st_ref = (kmc_b200.SignatureStats(k, m, max_batch_bytes=cap) for _ in range(2))
    half = len(data) // 2
    c1 = st.add_fastx(p, data[:half], False)
    st.add_fastx(p, data[c1:], True)
    st_ref.add(batch)
    assert np.array_equal(st.read(), st_ref.read())
    sk, sk_ref = (kmc_b200.SmallKCounter(11, not orig, max_batch_bytes=cap) for _ in range(2))
    assert sk.add_fastx(p, data, True) == len(data) and sk.last_seq_bytes == batch.size
    sk_ref.add(batch)
    assert np.array_equal(sk.read(), sk_ref.read())
    est, est_ref = (kmc_b200.HistogramEstimator(25, 7, max_batch_bytes=cap) for _ in range(2))
    assert est.add_fastx(p, data, True) == len(data)
    assert est.last_records == int(np.count_nonzero(batch == 10))
    est_ref.add(batch)
    assert np.array_equal(est.histogram(), est_ref.histogram())
    for x in (p, sp, ref, st, st_ref, sk, sk_ref, est, est_ref):
        x.close()


# ----------------------------------------------------------------------------- files -> databases
GOLDEN = json.load(open(BAM_GOLDEN))


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def _run_case(name, path, out, parse, batch_bytes=1 << 26):
    from kmc_b200 import reads
    k, opts, kw = BAM_CASES[name]
    if "-e" in opts:
        reads.write_histogram(out + ".txt", reads.estimate_histogram([path], k, batch_bytes=batch_bytes, parse=parse))
        return {"histogram_md5": md5(out + ".txt")}
    res = reads.count_reads([path], out, k, 9, None, batch_bytes=batch_bytes, parse=parse, **kw)
    return {"kmc_pre_md5": md5(out + ".kmc_pre"), "kmc_suf_md5": md5(out + ".kmc_suf"), "unique_kmers": res["n_unique"],
            "total_kmers": res["n_total"], "counted_kmers": res["n_unique"] - res["n_cutoff_min"] - res["n_cutoff_max"]}


def _expected(name):
    g = GOLDEN[name]
    return {key: g[key] for key in ("histogram_md5", "kmc_pre_md5", "kmc_suf_md5", "unique_kmers", "total_kmers", "counted_kmers") if key in g}


@pytest.fixture(scope="module")
def case_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("bam")
    return {layout: write(str(d / ("in_%s.bam" % layout)), case_bam(layout)[0]) for layout in ("aligned", "fixed", "random")}


@pytest.mark.parametrize("parse", ["gpu", "host"])
@pytest.mark.parametrize("name", sorted(BAM_CASES))
def test_bam_input_gives_the_reference_files(tmp_path, case_files, name, parse):
    assert _run_case(name, case_files["aligned"], str(tmp_path / "db"), parse) == _expected(name)


@pytest.mark.parametrize("batch_bytes", [(1 << 17) + 2, 1 << 20])
@pytest.mark.parametrize("layout", ["fixed", "random"])
def test_every_layout_and_small_pieces_give_the_reference_files(tmp_path, case_files, layout, batch_bytes):
    """Pieces of 64 KiB of text: the header spans several pieces, records straddle every piece."""
    for name in ("k31_b", "k11_small", "k31_e"):
        assert _run_case(name, case_files[layout], str(tmp_path / name), "gpu", batch_bytes) == _expected(name), name


def test_stage0_sample_ends_on_a_record_of_the_budget(tmp_path, monkeypatch):
    """With a small sample budget, the GPU reader's limit and the host model cut the records at the same place."""
    from kmc_b200 import reads
    monkeypatch.setattr(reads, "STATS_SAMPLE_BYTES", 300_000)
    raw, _ = case_bam("random")
    path = write(str(tmp_path / "in.bam"), raw)
    host = reads.signature_sample_counts([path], 31, 9, batch_bytes=1 << 20, parse="host")
    gpu = reads.signature_sample_counts([path], 31, 9, batch_bytes=1 << 20, parse="gpu")
    assert np.array_equal(host, gpu) and host.sum() > 0


def test_bad_files_are_errors_on_the_gpu_path(tmp_path):
    import gzip
    import kmc_b200
    from kmc_b200 import reads
    raw, text = bam_file(header(), odd_records(13, 40), "fixed")
    for name, data in [("no_eof", raw[:-28]), ("not_bgzf", gzip.compress(text) + raw[-28:])]:
        path = write(str(tmp_path / (name + ".bam")), data)
        assert reads.is_bam(path)
        with pytest.raises(kmc_b200.KmcB200Error) as e:
            reads.count_reads([path], str(tmp_path / name), 31, 9, None, parse="gpu")
        assert e.value.code == kmc_b200.ERR_INVALID, name


# ----------------------------------------------------------------------------- record counts past 2^24 in one chunk
def tiny_records(n):
    """n records of 39 bytes (one base, a NUL name, no CIGAR): every 7th from the 4th on secondary, every 5th FLAG 0x10, bases A C G in turn.
    Returns the bytes and the batch KMCB200_BAM_ORIGINAL_STRAND makes of them."""
    i = np.arange(n)
    rec = np.zeros(n, dtype=[("bs", "<i4"), ("ref", "<i4"), ("pos", "<i4"), ("l_name", "u1"), ("mapq", "u1"), ("bin", "<u2"),
                             ("n_cigar", "<u2"), ("flag", "<u2"), ("l_seq", "<i4"), ("nref", "<i4"), ("npos", "<i4"), ("tlen", "<i4"),
                             ("name", "u1"), ("seq", "u1"), ("qual", "u1")])
    rec["bs"], rec["ref"], rec["pos"], rec["l_name"], rec["l_seq"], rec["nref"], rec["npos"] = 35, -1, -1, 1, 1, -1, -1
    rec["flag"] = np.where(i % 5 == 0, 0x10, 0) | np.where(i % 7 == 3, 0x100, 0)
    rec["seq"] = np.array([1, 2, 4], dtype=np.uint8)[i % 3] << 4
    kept = i % 7 != 3
    base = np.frombuffer(b"ACG", dtype=np.uint8)[i % 3]
    base = np.where(i % 5 == 0, np.frombuffer(b"TGC", dtype=np.uint8)[i % 3], base)[kept]
    want = np.empty(2 * base.size, dtype=np.uint8)
    want[0::2], want[1::2] = base, 10
    return rec.tobytes(), want


def test_more_than_2_24_kept_records_in_one_chunk():
    """A chunk of 2^24 + 1000 kept records (the smallest records there are): the record table, the result words and the decode hold
    every record count a chunk of up to 2^31 bytes can have."""
    import kmc_b200
    n = (((1 << 24) + 1000) * 7) // 6 + 7
    data, want = tiny_records(n)
    assert want.size // 2 > (1 << 24) + 1000
    head = 5000 * 39
    assert _batch(data[:head], True) == tiny_records(5000)[1].tobytes()     # the generator's batch is the model's
    p = parser(kmc_b200.BAM_ORIGINAL_STRAND, max_chunk=len(data))
    seq, c = p.parse(data, True)
    assert c == len(data) and p.last_records() == want.size // 2
    assert seq.size == want.size and np.array_equal(seq, want)
    p.close()


def test_members_with_other_extra_subfields_on_both_paths(tmp_path):
    from bam_testlib import bgzf_member_extra
    from gzip_testlib import BGZF_EOF
    from kmc_b200 import reads
    _, text = case_bam()
    raw = b"".join(bgzf_member_extra(text[i:i + 60000]) for i in range(0, len(text), 60000)) + BGZF_EOF
    path = write(str(tmp_path / "extra.bam"), raw)
    for parse in ("gpu", "host"):
        res = reads.count_reads([path], str(tmp_path / parse), 31, 9, None, parse=parse)
        assert {"kmc_pre_md5": md5(str(tmp_path / parse) + ".kmc_pre"), "kmc_suf_md5": md5(str(tmp_path / parse) + ".kmc_suf"),
                "unique_kmers": res["n_unique"]} == {k: GOLDEN["k31"][k] for k in ("kmc_pre_md5", "kmc_suf_md5", "unique_kmers")}, parse
