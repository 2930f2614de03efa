"""CPU: the seam builder of tests/seam_testlib.py does what tests/test_gpu_seams.py relies on.  A planted m-mer gives a run of exactly
w = k - m + 1 k-mers where it was planted, poly-A segments give runs and records of the lengths asked for, and the numpy record model
agrees with the stage-1 oracle record for record."""
import numpy as np
import pytest

from seam_testlib import (FASTX_SPAN, FASTX_TILE, PACK_WINDOW, TILE, SeamBatch, check_line_ends, kmer_signatures, norm_table, offsets,
                          poly_a_segment, record_bytes, records_batch, runs, sampled_kmers, seam_anchors, sizes_to, super_kmers,
                          text_with_line_ends)
from stage1_testlib import Stage1Oracle, records


def oracle_record_lengths(batch, k, m):
    """k-mers per record, in input order, from the oracle's one-bin split"""
    sp = Stage1Oracle().split(batch, k, m, np.zeros((1 << (2 * m)) + 1, np.uint32), 1)
    return np.array([a + 1 for a, _ in records(sp.bin_data(0), k)], dtype=np.int64)


@pytest.mark.parametrize("k,m", [(6, 5), (31, 9), (12, 11), (33, 11), (128, 5)])
def test_planted_mmer_gives_a_run_of_exactly_w_kmers(k, m):
    b = SeamBatch(3 * TILE + 77, seed=k * 31 + m)
    want = []
    for j, a in seam_anchors(len(b), 256, margin=2):
        if a + 256 + k < len(b):
            b.plant_run(a + offsets(j), k, m)
            want.append(a + offsets(j))
    sig = kmer_signatures(b.a, k, m, norm_table(m))
    rs, re = runs(sig)
    w = k - m + 1
    for t in want:
        i = np.searchsorted(rs, t)
        assert rs[i] == t and re[i] == t + w - 1 and sig[t] < 4 ** (m - 1), t
    s, e = super_kmers(sig)
    assert np.array_equal(e - s + 1, oracle_record_lengths(b.tobytes(), k, m))


@pytest.mark.parametrize("k,m", [(31, 9), (128, 11)])
def test_poly_a_runs_and_separators(k, m):
    b = SeamBatch(24 * TILE, seed=5)
    want = []
    for i, n in enumerate((255, 256, 257, 511, 512, 513) * 3):
        end = (i + 1) * TILE + offsets(i)
        b.poly_a(end - n + 1, n, k)
        want.append((end - n + 1, end))
    b.lower(10, 20)
    sig = kmer_signatures(b.a, k, m, norm_table(m))
    rs, re = runs(sig)
    s, e = super_kmers(sig)
    for lo, hi in want:
        assert (lo, hi) in set(zip(rs.tolist(), re.tolist()))
        assert sig[lo] == 4 ** m
        cuts = set(s.tolist())
        assert all(t in cuts for t in range(lo, hi + 1, 256)) and hi in set(e.tolist())
    assert np.array_equal(e - s + 1, oracle_record_lengths(b.tobytes(), k, m))


def test_records_of_chosen_sizes():
    k = 128
    for nbytes in range(33, 98):
        seg = poly_a_segment(nbytes, k)
        s, e = super_kmers(kmer_signatures(np.frombuffer(seg, np.uint8), k, 5, norm_table(5)))
        assert s.size == 1 and record_bytes(s, e, k)[0] == nbytes
    sizes = sizes_to(PACK_WINDOW - 1, 33) + [50]
    sp = Stage1Oracle().split(records_batch(sizes, k), k, 5, np.zeros(4 ** 5 + 1, np.uint32), 1)
    assert int(sp.frags[0][3]) == len(sizes) and int(sp.frags[0][1]) == sum(sizes)
    assert list(sp.pack_bytes) == [PACK_WINDOW - 1 + 50]       # the record that starts at W - 1 is in pack 0
    for total in (33, 96, 97, 98, 1000, PACK_WINDOW):
        z = sizes_to(total, 33)
        assert sum(z) == total and all(33 <= x <= 97 for x in z)


@pytest.mark.parametrize("fmt", ["fastq", "fasta"])
def test_line_ends_land_on_the_seams(fmt):
    targets = []
    for j, a in seam_anchors(6 * FASTX_TILE, FASTX_SPAN * 37, margin=8):
        kinds = ("lf", "crlf", "hdr") if fmt == "fasta" else ("lf", "crlf")
        targets.append((kinds[j % len(kinds)], a + (j // len(kinds)) % 2 - 1))
    for t in range(1, 6):
        targets.append(("lf", t * FASTX_TILE - 1))
        targets.append(("crlf", t * FASTX_TILE + 4000))
    text, placed = text_with_line_ends(fmt, targets, 6 * FASTX_TILE, seed=3)
    check_line_ends(text, placed)
    assert len(placed) >= 0.9 * len(targets)


def test_sampled_kmers_are_sampled():
    from estimate_testlib import oracle_increments
    for k in (31, 64):
        kms = sampled_kmers(k, 7, 3, seed=k)
        assert len(kms) == 3 and all(oracle_increments(x, k, 7).size for x in kms)
    assert sampled_kmers(1, 7, 1, seed=1, max_tries=100) == []         # neither 1-mer (A/T, C/G) is sampled at s = 7
