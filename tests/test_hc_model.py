"""CPU: the batch rule of homopolymer compression (hc_testlib.homopolymer_compress, the rule the GPU applies) against a per-read
transcription of the reference's HomopolymerCompressSeq, and, through the stage-1 / stage-2 oracles and the small-k model, against what
the unmodified reference CLI wrote with `-hc -sr1` (tests/golden/hc_reference.json, made by tests/golden/make_hc_reference.py)."""
import hashlib
import os

import numpy as np
import pytest

from hc_testlib import HC_CASES, case_format, case_reads, compress_read, golden, homopolymer_compress, load_map, make_hc_reads, option, padded, \
    write_case_input
from kmc_b200.reads import sequences_to_batch
from kmc_testlib import Params, digest
from stage1_testlib import Stage1Oracle, batch_of
from test_small_k_model import counts, database, kmer_values

BIN_CASES = [n for n, c in HC_CASES.items() if c[4] > 13 and "-e" not in c[5]]
SMALL_CASES = [n for n, c in HC_CASES.items() if c[4] <= 13]


def md5(b):
    return hashlib.md5(b).hexdigest()


def case_batch(name, tmp):
    path = os.path.join(str(tmp), name + ".input")
    write_case_input(name, path)
    data = open(path, "rb").read()
    assert md5(data) == golden()[name]["input_md5"], "the generated input is not the one the reference counted"
    return sequences_to_batch(data)


def test_rule_on_short_inputs():
    assert homopolymer_compress(b"AAACCgGGTtaA\nAAcNNNNaa").tobytes() == b"ACgTa\nAcNNNNa"
    assert compress_read(b"AAACCgGGTtaANNNNRRaa") == b"ACgTaNa"
    assert homopolymer_compress(b"").size == 0 and homopolymer_compress(b"a").tobytes() == b"a"
    assert padded(b"AAAA\nCC").tobytes() == b"A\nC\n\n\n\n"
    assert homopolymer_compress(b"\n\n\r\rNN").tobytes() == b"\n\n\r\rNN"              # non-ACGT bytes are never dropped


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("k", [1, 5, 11, 21, 31])
def test_batch_rule_equals_the_per_read_rule(seed, k):
    """The k-mers (both strands and as they are) of the batch rule over the joined reads are the k-mers of the reads compressed one at a
    time as the reference does, for every k; the padding changes nothing."""
    reads = make_hc_reads(seed, "hp", 400, 300, k)
    batch = batch_of(reads)
    per_read = batch_of([compress_read(r) for r in reads])
    for both in (True, False):
        want = np.sort(kmer_values(np.frombuffer(per_read, dtype=np.uint8), k, both))
        assert np.array_equal(np.sort(kmer_values(homopolymer_compress(batch), k, both)), want)
        assert np.array_equal(np.sort(kmer_values(padded(batch), k, both)), want)


def test_generated_reads_hold_what_they_promise():
    k = 31
    reads = make_hc_reads(7, "hp", 800, 300, k)
    lens = {len(compress_read(r)) for r in reads[4::8]}
    assert {k - 1, k, k + 1} <= lens                                   # reads that compress to k - 1, k, k + 1 bases
    assert any(len(set(r.upper())) == 1 and len(r) > 1 for r in reads)  # one base repeated
    assert any(b"aA" in r or b"Aa" in r for r in reads)                 # mixed-case runs
    assert any(b"AN" in r or b"NA" in r for r in reads)                 # runs next to N
    assert any(reads[i][-1:].upper() == reads[i + 1][:1].upper() for i in range(5, len(reads) - 1, 8))   # a run across a read boundary
    assert max(len(r) - len(compress_read(r)) for r in reads) >= 250


def test_golden_cases_are_the_declared_ones():
    g = golden()
    assert sorted(g) == sorted(HC_CASES)
    for name in SMALL_CASES:
        assert g[name]["version"] == 0, "the reference did not take its small-k path"


@pytest.mark.parametrize("case", BIN_CASES)
def test_oracle_on_the_compressed_batch_equals_kmc_hc(tmp_path, case, oracle):
    """oracle split of homopolymer_compress(batch) -> oracle stage 2 -> per file-bin payload / LUT digests equal `kmc -hc`'s database;
    the k-mers and super-k-mers add up to the reference's totals."""
    c = golden()[case]
    batch = homopolymer_compress(case_batch(case, tmp_path))
    h = c["header"]
    n_bins = len(c["bins"])
    sp = Stage1Oracle().split(batch.tobytes(), h["k"], h["sig_len"], load_map(case), n_bins)
    p = Params(k=h["k"], both_strands=h["both"], cutoff_min=h["cmin"], cutoff_max=h["cmax"], counter_max=c["counter_max"], lut_prefix_len=h["p"])
    for b in range(n_bins):
        r = oracle.process_bin(sp.to_bin(b), p)
        assert {"payload": digest(r.payload), "lut": digest(np.asarray(r.lut, dtype=np.uint64))} == c["bins"][b], "bin %d" % b
    assert int(sp.frags[:, 2].sum()) == c["total_kmers"]
    assert int(sp.frags[:, 3].sum()) == c["total_super_kmers"]


@pytest.mark.parametrize("case", SMALL_CASES)
def test_small_k_model_on_the_compressed_batch_equals_kmc_hc(tmp_path, case):
    c = golden()[case]
    k = HC_CASES[case][4]
    both = "-b" not in HC_CASES[case][5]
    cmin, cmax, cs = option(case, "-ci", 2), option(case, "-cx", 1_000_000_000), option(case, "-cs", 255)
    pre, suf, stats, lp = database(counts(homopolymer_compress(case_batch(case, tmp_path)), k, both), k, both, cmin, cmax, cs)
    assert stats[3] == c["total_kmers"] and stats[0] == c["unique_kmers"] and lp == c["lut_prefix_len"]
    assert md5(pre) == c["kmc_pre_md5"] and md5(suf) == c["kmc_suf_md5"]


def test_uncompressed_model_differs_from_kmc_hc(tmp_path):
    """The stored databases are compressed ones: the same model without compression does not give them."""
    case = "k5_small"
    pre, suf, stats, _ = database(counts(case_batch(case, tmp_path), 5), 5, True, 1, 1_000_000_000, 255)
    assert stats[3] != golden()[case]["total_kmers"]


def test_formats_of_the_cases():
    assert case_format("k31_p9_fa") == "-fa" and case_format("k31_p9_fm") == "-fm" and case_format("k31_p9") == "-fq"
    assert len(case_reads("k31_p9")) == HC_CASES["k31_p9"][2]
