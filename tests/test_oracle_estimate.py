"""The histogram estimator's oracle (oracle/estimate_oracle.c) against the reference: every stored `kmc -e` file and every stored result of the
reference's CntHashEstimator (tests/golden/estimate_reference.json), the reference's estimator itself where build() compiled it, and the
LUT prefix length rule of `kmc` / `kmc --opt-out-size`.  No GPU."""
import numpy as np
import pytest

import estimate_testlib as et
from kmc_b200.reads import estimated_counted_kmers, kmc_lut_prefix_len, n_records

GOLDEN = et.load_golden()


@pytest.mark.parametrize("case", [c for c in GOLDEN["cli"] + GOLDEN["harness"] if c["md5"]], ids=lambda c: c["name"])
def test_oracle_reproduces_the_reference(case):
    hist = et.oracle_histogram(et.case_batch(case), case["k"], case["s"])
    assert hist[0] == 0
    assert et.md5(et.hist_text(hist)) == case["md5"]


@pytest.mark.parametrize("k,s", [(1, 7), (9, 7), (31, 11), (64, 7), (129, 11), (256, 7)])
def test_oracle_equals_the_reference_estimator(k, s):
    if not et.have_harness():
        pytest.skip("oracle/_ref/libkmc_nthash_ref.so not built (the reference tree is absent)")
    batch = et.case_batch({"gen": {"kind": "reads", "seed": 77 + k, "n_reads": 150, "read_len": [50, 400], "lower_frac": 0.1}})
    assert np.array_equal(et.oracle_histogram(batch, k, s), et.harness_histogram(batch, k, s))


def test_oracle_increments_ignore_case_and_separators():
    reads = et.make_reads(5, 50, 300, n_frac=0.01)
    upper = b"".join(r + b"\n" for r in reads)
    mixed = b"".join(r.lower() + b"\r\n" if i % 2 else r + b"x" for i, r in enumerate(reads))
    a, b = et.oracle_increments(upper, 25, 7), et.oracle_increments(mixed, 25, 7)
    assert a.size > 0 and np.array_equal(np.sort(a), np.sort(b))


def test_lut_prefix_len_rule():
    # k = 30, 64 bins: 4 * n_reads of 100 000 reads picks 2; the reference's estimate of the stored case picks 6
    case = next(c for c in GOLDEN["db"] if c["name"] == "lp_changes_k30")
    assert kmc_lut_prefix_len(30, 4 * case["gen"]["n_reads"], 64) == 2
    hist = et.oracle_histogram(et.case_batch(case), 30, 7)
    assert kmc_lut_prefix_len(30, estimated_counted_kmers(hist, 1, 1_000_000_000), 64) == 6
    assert kmc_lut_prefix_len(31, 0, 512) == 3                          # no k-mers: the smallest LUT


def test_n_records():
    reads = et.make_reads(3, 40, [50, 200])
    assert n_records(et.fastq_text(reads)) == 40
    assert n_records(et.fasta_multiline_text(reads)) == 40
    assert n_records(b"") == 0
