"""GPU: stage 0 on the H100 — signature statistics (kmcb200_sigstats_* / kmcb200_dev_sigstats_add) against the oracle's literal CalcStats,
the splitter's opt-in (k+x)-mer totals against the oracle's collector rule, and reads -> database with the map chosen from the reads against
the reference CLI's stored and live results."""
import os

import numpy as np
import pytest

from stage0_testlib import max_x_of, oracle_kxmer_totals, oracle_signature_stats
from stage1_testlib import STAGE1_CASES, STAGE1_GOLDEN, Split, Stage1Oracle, batch_of, case_reads, make_reads, random_map, write_fastq_reads

pytestmark = pytest.mark.gpu

PROFILES = {"short": (40, 150), "long": (6, 10_000), "n_dense": (60, 200), "low_complexity": (8, 3000)}


@pytest.fixture(scope="module")
def s1():
    return Stage1Oracle()


def profile_batch(seed):
    reads = []
    for j, (prof, (n, ln)) in enumerate(PROFILES.items()):
        reads += make_reads(seed + j, prof, n_reads=n, read_len=ln)
    return batch_of(reads)


def matrix():
    return [(k, m) for m in (5, 9, 11) for k in sorted({m + 1, 17, 31, 32, 33, 64, 65, 127, 128})]


@pytest.mark.parametrize("k,m", matrix())
def test_counts_match_oracle(k, m):
    import kmc_b200
    batch = profile_batch(1000 * k + 10 * m)
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(batch))
    before = st.kernel_launches()
    st.add(batch)
    assert st.kernel_launches() - before == 1
    got = st.read()
    assert np.array_equal(got, oracle_signature_stats(batch, k, m))
    assert int(got.sum()) > 0
    st.close()


@pytest.mark.parametrize("k,m", [(31, 9), (128, 5), (12, 11)])
def test_one_read_of_five_million_bases(k, m):
    import kmc_b200
    rng = np.random.default_rng(k + m)
    read = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 5_000_000)].copy()
    read[rng.integers(0, read.size, 50)] = ord("N")
    read[1_000_000:1_300_000] = ord("A")                     # one run of far more than a warp's positions: the special signature
    batch = read.tobytes()
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(batch))
    st.add(batch)
    exp = oracle_signature_stats(batch, k, m)
    got = st.read()
    assert np.array_equal(got, exp)
    assert int(got[-1]) >= 300_000 - k
    st.close()


def test_batches_accumulate_and_reset():
    import kmc_b200
    k, m = 31, 9
    reads = make_reads(5, "short", 3000) + make_reads(6, "long", 20, 10_000) + make_reads(7, "low_complexity", 20, 3000)
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=1 << 24)
    st.add(batch_of(reads))
    whole = st.read()
    assert np.array_equal(whole, oracle_signature_stats(batch_of(reads), k, m))
    st.reset()
    assert not st.read().any()
    cuts = [0, 1, 700, 701, 2900, 3010, 3030, len(reads)]
    for a, b in zip(cuts[:-1], cuts[1:]):
        st.add(batch_of(reads[a:b]))
    assert np.array_equal(st.read(), whole)
    st.add(batch_of(reads))
    assert np.array_equal(st.read(), 2 * whole)
    st.close()


def test_device_twin_on_a_torch_stream():
    import torch
    import kmc_b200
    k, m = 33, 9
    batch = batch_of(make_reads(9, "short", 2000) + make_reads(10, "n_dense", 200))
    exp = oracle_signature_stats(batch, k, m)
    st = kmc_b200.SignatureStats(k, m, max_batch_bytes=len(batch))
    dev = torch.device("cuda:0")
    d_seq = torch.frombuffer(bytearray(batch), dtype=torch.uint8).to(dev)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    before = st.kernel_launches()
    with torch.cuda.stream(s):
        st.dev_add(d_seq.data_ptr(), len(batch), s.cuda_stream)
        st.dev_add(d_seq.data_ptr(), len(batch), s.cuda_stream)
    assert st.kernel_launches() - before == 2
    assert np.array_equal(st.read(), 2 * exp)                          # read waits for the stream's work
    st.reset()
    st.dev_add(d_seq.data_ptr(), len(batch), None)
    assert np.array_equal(st.read(), exp)
    st.close()


def test_empty_tiny_and_oversized_batches():
    import kmc_b200
    st = kmc_b200.SignatureStats(6, 5, max_batch_bytes=4096)
    total = np.zeros((1 << 10) + 1, dtype=np.uint32)
    for batch in (b"", b"\n", b"ACGTA", b"ACGTAC", b"NNNNNNNN", b"acgtacgtacgt\nAC", b"A" * 4096):
        st.add(batch)
        total += oracle_signature_stats(batch, 6, 5)
        assert np.array_equal(st.read(), total), batch[:20]
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        st.add(b"A" * 4097)
    assert ei.value.code == kmc_b200.ERR_INVALID
    assert np.array_equal(st.read(), total)
    st.close()
    for kw in (dict(kmer_len=5, signature_len=5), dict(kmer_len=129, signature_len=7), dict(kmer_len=31, signature_len=4),
               dict(kmer_len=31, signature_len=12), dict(max_batch_bytes=0), dict(max_batch_bytes=(1 << 31) + 1)):
        a = dict(kmer_len=31, signature_len=7, max_batch_bytes=1 << 20)
        a.update(kw)
        with pytest.raises(kmc_b200.KmcB200Error) as ei:
            kmc_b200.SignatureStats(a["kmer_len"], a["signature_len"], max_batch_bytes=a["max_batch_bytes"])
        assert ei.value.code == kmc_b200.ERR_INVALID, kw


# ----------------------------------------------------------------------------- (k+x)-mer totals of the splitter
def gpu_split(sp, batch) -> Split:
    out, packs, frags = sp.split_raw(batch)
    fr = np.array([[f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs] for f in frags], dtype=np.uint64)
    return Split(out.copy(), packs.copy(), fr, sp.kmer_len)


@pytest.mark.parametrize("k", [17, 31, 32, 55, 96])
@pytest.mark.parametrize("both", [True, False])
def test_splitter_kxmer_totals_match_oracle(s1, k, both):
    import kmc_b200
    m, n_bins = 9, 512
    sig_map = random_map(k, m, n_bins)
    reads = []
    for j, (prof, (n, ln)) in enumerate(PROFILES.items()):
        reads += make_reads(77 * k + j, prof, n_reads=n, read_len=ln)
    halves = (batch_of(reads[:50]), batch_of(reads[50:]))
    plain = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=1 << 22)
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=1 << 22)
    sp.count_kxmers(both)
    exp = np.zeros(n_bins, dtype=np.uint64)
    for batch in halves:
        b0, b1 = plain.kernel_launches(), sp.kernel_launches()
        want, got = gpu_split(plain, batch), gpu_split(sp, batch)
        extra = 1 if max_x_of(k) else 0                              # k = 31, 32: stage 2 sorts plain k-mers, nothing to count
        assert sp.kernel_launches() - b1 == plain.kernel_launches() - b0 + extra
        assert np.array_equal(got.frags, want.frags) and got.out.tobytes() == want.out.tobytes() and np.array_equal(got.pack_bytes, want.pack_bytes)
        exp += oracle_kxmer_totals(s1.split(batch, k, m, sig_map, n_bins), both)
    assert np.array_equal(sp.kxmer_totals(), exp)
    assert (int(exp.sum()) > 0) == bool(max_x_of(k))
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        plain.kxmer_totals()
    assert ei.value.code == kmc_b200.ERR_INVALID
    sp.count_kxmers(both)                                               # enabling again zeroes the totals
    assert not sp.kxmer_totals().any()
    sp.close()
    plain.close()


def test_capacity_error_adds_no_kxmers(s1):
    import torch
    import kmc_b200
    k, m, n_bins = 29, 7, 64
    sig_map = random_map(4, m, n_bins)
    batch = batch_of(make_reads(12, "short", 500))
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch))
    sp.count_kxmers(True)
    exp = oracle_kxmer_totals(s1.split(batch, k, m, sig_map, n_bins), True)
    dev = torch.device("cuda:0")
    d_seq = torch.frombuffer(bytearray(batch), dtype=torch.uint8).to(dev)
    d_frags = torch.zeros(n_bins * 5, dtype=torch.int64, device=dev)
    d_res = torch.zeros(8, dtype=torch.int64, device=dev)
    sp.dev_split(d_seq.data_ptr(), len(batch), 0, 0, 0, 0, d_frags.data_ptr(), d_res.data_ptr(), None)   # sizing only: capacity flag
    torch.cuda.synchronize()
    assert int(d_res[2]) == 1
    assert not sp.kxmer_totals().any()
    sp.split_raw(batch)
    assert np.array_equal(sp.kxmer_totals(), exp)
    sp.close()


# ----------------------------------------------------------------------------- reads -> database, map chosen from the reads
def _golden_case(case):
    import json
    return json.load(open(STAGE1_GOLDEN))["cases"][case]


@pytest.mark.parametrize("case", sorted(STAGE1_CASES))
def test_count_reads_without_a_map_matches_stored_reference_database(tmp_path, case):
    from kmc_b200.reads import count_reads
    from kmc_testlib import digest
    c = _golden_case(case)
    h = c["header"]
    fq = str(tmp_path / "reads.fq")
    write_fastq_reads(fq, case_reads(case))
    out = str(tmp_path / "db")
    res = count_reads([fq], out, h["k"], h["sig_len"], None, h["p"], h["cmin"], h["cmax"], c["counter_max"], h["both"], batch_bytes=1 << 20,
                      n_bins=len(c["bins"]))
    assert {ext: digest(open(out + ext, "rb").read()) for ext in (".kmc_pre", ".kmc_suf")} == c["files"]
    assert res["n_kmers"] == c["total_kmers"] == res["n_total"]
    assert res["n_super_kmers"] == c["total_super_kmers"]


def test_cli_without_a_map(tmp_path):
    import subprocess
    import sys
    from kmc_testlib import digest
    case = "k55_p9_ndense_b"
    c = _golden_case(case)
    h = c["header"]
    fq = str(tmp_path / "reads.fq")
    write_fastq_reads(fq, case_reads(case))
    out = str(tmp_path / "db")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run([sys.executable, "-m", "kmc_b200.reads", "-n64", "-k%d" % h["k"], "-p%d" % h["sig_len"], "--lut-prefix-len", str(h["p"]),
                    "--ci", str(h["cmin"]), "--cs", str(c["counter_max"]), "-b", fq, out], check=True, cwd=root, capture_output=True)
    assert {ext: digest(open(out + ext, "rb").read()) for ext in (".kmc_pre", ".kmc_suf")} == c["files"]


@pytest.mark.parametrize("k", [17, 31, 55])
@pytest.mark.parametrize("p", [7, 9, 11])
@pytest.mark.parametrize("both", [True, False])
def test_count_reads_without_a_map_matches_reference_cli(tmp_path, k, p, both):
    """Where the reference CLI is built: the same FASTQ through kmc_ref -sr1 (default -n) and through count_reads with no map."""
    from kmc_b200.reads import count_reads
    from test_gpu_kmc_files import KMC_REF, count, md5
    if not os.path.exists(KMC_REF):
        pytest.skip("oracle/_ref/kmc_ref not built")
    tmp = str(tmp_path)
    fq = os.path.join(tmp, "reads.fq")
    write_fastq_reads(fq, make_reads(7 * k + p, "short", 20000, 150, genome_len=300_000) + make_reads(p, "n_dense", 2000, 150))
    ref_db, st = count(KMC_REF, tmp, "ref", fq, k, ("-p%d" % p, "-ci2", "-sr1") + (() if both else ("-b",)))
    from stage1_testlib import kmc_pre_bins
    h = kmc_pre_bins(ref_db + ".kmc_pre", ref_db + ".kmc_suf")[0]
    out = os.path.join(tmp, "gpu")
    res = count_reads([fq], out, k, p, None, h["p"], h["cmin"], h["cmax"], 255, both, batch_bytes=1 << 21)
    assert md5(out + ".kmc_suf") == md5(ref_db + ".kmc_suf")
    assert md5(out + ".kmc_pre") == md5(ref_db + ".kmc_pre")
    s = st.get("Stats", st)
    assert res["n_super_kmers"] == int(s["#Total_super-k-mers"])
