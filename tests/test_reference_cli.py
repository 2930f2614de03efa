"""BASELINE configs[0] (CPU plumbing, no GPU): a ~1 MB synthetic FASTQ through the UNMODIFIED reference CLI at k = 15 (the regular bin
pipeline: the small-k direct-count path needs k <= 13, SURVEY section 0.2) and k = 13 (small-k path), checked against a brute-force count of
the reads (the reference's own test strategy: tests/kmc_CLI/trivial-k-mer-counter).  This pins the test infrastructure the whole-file GPU
parity tests rest on (the FASTQ writer, the brute-force counter, the dump format).  What the reference CLI counted (`kmc -ci2 -cs255`, then
`kmc_tools transform ... dump -s`) is stored as a digest of its sorted dump in tests/golden/reference_digests.json
(tests/golden/make_reference_digests.py), so the test needs no reference build."""
import os

import pytest

from kmc_testlib import digest, reference_digest
from test_gpu_kmc_files import write_fastq

CLI_KS = [15, 13]


def brute_force(fastq, k, both=True):
    comp = {"A": "T", "C": "G", "G": "C", "T": "A"}
    cnt = {}
    with open(fastq) as f:
        for i, line in enumerate(f):
            if i % 4 != 1:
                continue
            for piece in line.strip().split("N"):
                for j in range(len(piece) - k + 1):
                    km = piece[j:j + k]
                    if both:
                        rc = "".join(comp[c] for c in reversed(km))
                        km = min(km, rc)
                    cnt[km] = cnt.get(km, 0) + 1
    return cnt


def small_fastq(path):
    write_fastq(path, 15, 3400, genome_len=200_000)          # 3400 x 150 bp: ~1 MB of FASTQ


def dump_digest(counts):
    """A k-mer -> count map in the form `kmc_tools transform ... dump -s` prints it (sorted 'kmer<TAB>count' lines), as a digest."""
    return digest("".join("%s\t%d\n" % (km, c) for km, c in sorted(counts.items())).encode())


@pytest.mark.parametrize("k", CLI_KS)
def test_reference_cli_on_a_small_fastq(tmp_path, k):
    fq = os.path.join(str(tmp_path), "reads.fq")
    small_fastq(fq)
    assert 0.9e6 < os.path.getsize(fq) < 1.3e6
    ref = reference_digest("cli_fastq_k%d" % k)
    assert digest(open(fq, "rb").read()) == ref["input"], "the generated FASTQ is not the one the reference counted"
    exp = {km: min(c, 255) for km, c in brute_force(fq, k).items() if c >= 2}
    assert dump_digest(exp) == ref["results"]["dump"]
    assert ref["results"]["unique_counted_kmers"] == len(exp)
