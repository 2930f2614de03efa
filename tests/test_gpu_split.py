"""GPU: stage 1 on the H100 (kmcb200_split / kmcb200_dev_split) against the sequential C oracle byte for byte, against stored results of
the unmodified reference CLI, and straight into stage 2."""
import ctypes as C
import os

import numpy as np
import pytest

from stage1_testlib import (STAGE1_CASES, Split, Stage1Oracle, batch_of, case_reads, concat_splits, kmc_pre_bins, load_map, make_reads,
                            random_map, write_fastq_reads)

pytestmark = pytest.mark.gpu

PROFILES = {"short": (40, 150), "long": (6, 10_000), "n_dense": (60, 200), "low_complexity": (8, 3000)}


@pytest.fixture(scope="module")
def s1():
    return Stage1Oracle()


def gpu_split(sp, batch) -> Split:
    out, packs, frags = sp.split_raw(batch)
    fr = np.array([[f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs] for f in frags], dtype=np.uint64)
    return Split(out.copy(), packs.copy(), fr, sp.kmer_len)


def assert_same(got: Split, exp: Split):
    assert np.array_equal(got.frags, exp.frags)
    assert got.out.tobytes() == exp.out.tobytes()
    assert np.array_equal(got.pack_bytes, exp.pack_bytes)


def matrix():
    cases = []
    for m in (5, 9, 11):
        for i, k in enumerate(sorted({m + 1, 17, 31, 32, 33, 64, 65, 127, 128})):
            cases.append((k, m, (64, 512, 4096)[(i + m) % 3]))
    return cases


@pytest.mark.parametrize("k,m,n_bins", matrix())
def test_gpu_matches_oracle(s1, k, m, n_bins):
    import kmc_b200
    sig_map = random_map(k * 131 + m, m, n_bins)
    reads = []
    for j, (prof, (n, ln)) in enumerate(PROFILES.items()):
        reads += make_reads(1000 * k + 10 * m + j, prof, n_reads=n, read_len=ln)
    batch = batch_of(reads)
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch) + 10)
    before = sp.kernel_launches()
    got = gpu_split(sp, batch)
    assert sp.kernel_launches() - before >= 10
    assert_same(got, s1.split(batch, k, m, sig_map, n_bins))
    assert np.all(got.pack_bytes <= 65536) and np.all(got.pack_bytes > 0)
    sp.close()


@pytest.mark.parametrize("k,m", [(31, 9), (128, 5), (12, 11)])
def test_one_read_of_five_million_bases(s1, k, m):
    import kmc_b200
    rng = np.random.default_rng(k + m)
    read = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 5_000_000)].copy()
    read[rng.integers(0, read.size, 50)] = ord("N")
    read[1_000_000:1_300_000] = ord("A")                     # one run of far more than 256 k-mers inside the read
    batch = read.tobytes()
    sig_map = random_map(7, m, 512)
    sp = kmc_b200.Splitter(k, m, sig_map, 512, max_batch_bytes=len(batch))
    assert_same(gpu_split(sp, batch), s1.split(batch, k, m, sig_map, 512))
    sp.close()


def test_batches_are_independent(s1):
    import kmc_b200
    k, m, n_bins = 31, 9, 512
    reads = make_reads(5, "short", 3000) + make_reads(6, "long", 20, 10_000) + make_reads(7, "low_complexity", 20, 3000)
    sig_map = random_map(11, m, n_bins)
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=1 << 24)
    whole = gpu_split(sp, batch_of(reads))
    cuts = [0, 1, 700, 701, 2900, 3010, 3030, len(reads)]
    parts = concat_splits([gpu_split(sp, batch_of(reads[a:b])) for a, b in zip(cuts[:-1], cuts[1:])])
    assert len(cuts) - 1 == 7
    for b in range(n_bins):
        assert parts.bin_data(b).tobytes() == whole.bin_data(b).tobytes()
        assert np.array_equal(parts.frags[b][1:4], whole.frags[b][1:4])
    # the pack lists concatenate too: each batch's fragment starts its own packs, which the oracle splits the same way
    exp = concat_splits([s1.split(batch_of(reads[a:b]), k, m, sig_map, n_bins) for a, b in zip(cuts[:-1], cuts[1:])])
    assert np.array_equal(parts.pack_bytes, exp.pack_bytes) and np.array_equal(parts.frags, exp.frags)
    sp.close()


def test_device_path_matches_host_path():
    import torch
    import kmc_b200
    k, m, n_bins = 33, 9, 512
    sig_map = random_map(3, m, n_bins)
    batch = batch_of(make_reads(9, "short", 2000) + make_reads(10, "n_dense", 200))
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch))
    host = gpu_split(sp, batch)
    dev = torch.device("cuda:0")
    d_seq = torch.frombuffer(bytearray(batch), dtype=torch.uint8).to(dev)
    d_out = torch.full((host.out.size + 64,), 0xAB, dtype=torch.uint8, device=dev)
    d_packs = torch.zeros(host.pack_bytes.size + 8, dtype=torch.int64, device=dev)
    d_frags = torch.zeros(n_bins * 5, dtype=torch.int64, device=dev)
    d_res = torch.zeros(8, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev)
    before = sp.kernel_launches()
    sp.dev_split(d_seq.data_ptr(), len(batch), d_out.data_ptr(), d_out.numel(), d_packs.data_ptr(), d_packs.numel(), d_frags.data_ptr(),
                 d_res.data_ptr(), stream.cuda_stream)
    torch.cuda.synchronize()
    assert sp.kernel_launches() - before >= 10
    res = d_res.cpu().numpy().astype(np.uint64)
    assert list(res[:5]) == [host.out.size, host.pack_bytes.size, 0, int(host.frags[:, 3].sum()), int(host.frags[:, 2].sum())]
    fr = d_frags.cpu().numpy().view(np.uint64).reshape(n_bins, 5)
    frags = np.concatenate([fr[:, :4], (fr[:, 4] & 0xFFFFFFFF)[:, None], (fr[:, 4] >> 32)[:, None]], axis=1)
    assert_same(Split(d_out.cpu().numpy()[:host.out.size], d_packs.cpu().numpy().view(np.uint64)[:host.pack_bytes.size], frags, k), host)
    # too small on the device: only the result words change
    d_out.fill_(0xCD)
    d_frags.fill_(-1)
    sp.dev_split(d_seq.data_ptr(), len(batch), d_out.data_ptr(), host.out.size - 1, d_packs.data_ptr(), d_packs.numel(), d_frags.data_ptr(),
                 d_res.data_ptr(), None)
    torch.cuda.synchronize()
    res = d_res.cpu().numpy().astype(np.uint64)
    assert list(res[:3]) == [host.out.size, host.pack_bytes.size, 1]
    assert bool((d_out == 0xCD).all()) and bool((d_frags == -1).all())
    sp.close()


def test_capacity_errors_and_retry():
    import kmc_b200
    k, m, n_bins = 31, 7, 64
    sig_map = random_map(4, m, n_bins)
    batch = batch_of(make_reads(12, "short", 500))
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch))
    exp_out, exp_packs, exp_frags = sp.split_raw(batch)
    exp_out, exp_packs = exp_out.copy(), exp_packs.copy()
    for ob, pb in ((exp_out.size - 1, exp_packs.size), (exp_out.size, exp_packs.size - 1), (0, 0)):
        out = np.full(max(ob, 1), 7, dtype=np.uint8)
        packs = np.full(max(pb, 1), 9, dtype=np.uint64)
        frags = (kmc_b200.BinFragment * n_bins)()
        nbytes, npacks = C.c_uint64(0), C.c_uint64(0)
        rc = sp.lib.kmcb200_split(sp._h, batch, len(batch), out.ctypes.data, ob, C.byref(nbytes), packs.ctypes.data, pb, C.byref(npacks), frags)
        assert rc == kmc_b200.ERR_CAPACITY
        assert (nbytes.value, npacks.value) == (exp_out.size, exp_packs.size)
        assert np.all(out == 7) and np.all(packs == 9) and all(f.bytes == 0 and f.n_rec == 0 for f in frags)
    out, packs, frags = sp.split_raw(batch, out=np.zeros(exp_out.size, np.uint8), pack_bytes=np.zeros(exp_packs.size, np.uint64))
    assert out.tobytes() == exp_out.tobytes() and np.array_equal(packs, exp_packs)
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        sp.split_raw(batch + b"\nACGT")                    # longer than max_batch_bytes
    assert ei.value.code == kmc_b200.ERR_INVALID
    sp.close()


def test_splitter_refuses_bad_maps_and_parameters():
    import kmc_b200
    good = random_map(1, 7, 64)
    for kw in (dict(kmer_len=7, signature_len=7), dict(kmer_len=129, signature_len=7), dict(kmer_len=31, signature_len=4, sig_map=random_map(1, 4, 64)),
               dict(kmer_len=31, signature_len=12, sig_map=np.zeros((1 << 24) + 1, np.uint32)), dict(n_bins=4097), dict(n_bins=0),
               dict(max_batch_bytes=0), dict(max_batch_bytes=(1 << 31) + 1)):
        a = dict(kmer_len=31, signature_len=7, sig_map=good, n_bins=64, max_batch_bytes=1 << 20)
        a.update(kw)
        with pytest.raises(kmc_b200.KmcB200Error) as ei:
            kmc_b200.Splitter(a["kmer_len"], a["signature_len"], a["sig_map"], a["n_bins"], max_batch_bytes=a["max_batch_bytes"])
        assert ei.value.code == kmc_b200.ERR_INVALID, kw
    bad = good.copy()
    bad[1234] = 64
    with pytest.raises(kmc_b200.KmcB200Error) as ei:
        kmc_b200.Splitter(31, 7, bad, 64)
    assert ei.value.code == kmc_b200.ERR_INVALID and "1234" in str(ei.value)
    with pytest.raises(kmc_b200.KmcB200Error):
        kmc_b200.Splitter(31, 7, good, 64, device=99)


def test_empty_and_tiny_batches(s1):
    import kmc_b200
    sig_map = random_map(2, 5, 64)
    sp = kmc_b200.Splitter(6, 5, sig_map, 64, max_batch_bytes=4096)
    for batch in (b"", b"\n", b"ACGTA", b"ACGTAC", b"NNNNNNNN", b"acgtacgtacgt\nAC"):
        assert_same(gpu_split(sp, batch), s1.split(batch, 6, 5, sig_map, 64))
    sp.close()


def test_split_bins_straight_into_stage2(s1, oracle):
    """GPU bins through process_bin and dev_process_bin equal the stage-2 oracle on the oracle's bins."""
    import torch
    import kmc_b200
    from kmc_testlib import Params, to_skb
    k, m, n_bins = 31, 9, 64
    sig_map = random_map(21, m, n_bins)
    batch = batch_of(make_reads(30, "short", 20000, genome_len=30_000) + make_reads(31, "low_complexity", 30, 3000))
    sp = kmc_b200.Splitter(k, m, sig_map, n_bins, max_batch_bytes=len(batch))
    got = gpu_split(sp, batch)
    exp = s1.split(batch, k, m, sig_map, n_bins)
    prm = Params(k=k, cutoff_min=2, lut_prefix_len=7)
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(k, True, 2, 10 ** 9, 255, 7))
    dev = torch.device("cuda:0")
    for b in range(0, n_bins, 3):
        e = oracle.process_bin(exp.to_bin(b), prm)
        r = ctx.process_bin(to_skb(got.to_bin(b)))
        assert r.stats == e.stats and r.payload.tobytes() == e.payload and np.array_equal(r.lut, e.lut), b
        gb = got.to_bin(b)
        d_bin = torch.zeros(gb.size + 64, dtype=torch.uint8, device=dev)
        d_bin[:gb.size] = torch.from_numpy(gb.data.copy()).to(dev)
        cap = ctx.out_capacity(gb.n_rec) + 64
        d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
        d_lut = torch.zeros(ctx.lut_entries, dtype=torch.int64, device=dev)
        d_res = torch.zeros(8, dtype=torch.int64, device=dev)
        ctx.dev_process_bin(0, d_bin.data_ptr(), gb.size, gb.n_rec, gb.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr())
        torch.cuda.synchronize()
        res = d_res.cpu().numpy()
        assert tuple(int(x) for x in res[:4]) == e.stats
        assert d_out.cpu().numpy()[:len(e.payload)].tobytes() == e.payload
        assert np.array_equal(d_lut.cpu().numpy().view(np.uint64), e.lut)
    ctx.close()
    sp.close()


# ----------------------------------------------------------------------------- whole databases against the reference CLI
@pytest.mark.parametrize("case", sorted(STAGE1_CASES))
def test_count_reads_matches_stored_reference_database(tmp_path, case):
    """count_reads with the map of the reference's .kmc_pre writes the same two files, byte for byte, as the reference CLI did (-sr1)."""
    import json
    from kmc_b200.reads import count_reads
    from kmc_testlib import digest
    from stage1_testlib import STAGE1_GOLDEN
    c = json.load(open(STAGE1_GOLDEN))["cases"][case]
    h = c["header"]
    fq = str(tmp_path / "reads.fq")
    write_fastq_reads(fq, case_reads(case))
    out = str(tmp_path / "db")
    res = count_reads([fq], out, h["k"], h["sig_len"], load_map(case), h["p"], h["cmin"], h["cmax"], c["counter_max"], h["both"], batch_bytes=1 << 20,
                      n_bins=len(c["bins"]))
    assert {ext: digest(open(out + ext, "rb").read()) for ext in (".kmc_pre", ".kmc_suf")} == c["files"]
    assert res["n_kmers"] == c["total_kmers"] == res["n_total"]
    assert res["n_super_kmers"] == c["total_super_kmers"]


REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")


@pytest.mark.parametrize("k", [17, 31, 55])
@pytest.mark.parametrize("p", [7, 9, 11])
@pytest.mark.parametrize("both", [True, False])
def test_count_reads_matches_reference_cli(tmp_path, k, p, both):
    """Where the reference CLI is built: the same FASTQ through kmc_ref -sr1 and through count_reads (map from its .kmc_pre)."""
    from kmc_b200.reads import count_reads, signature_map_from_kmc_pre
    from test_gpu_kmc_files import KMC_REF, KMC_TOOLS, count, dump_sorted, md5
    if not (os.path.exists(KMC_REF) and os.path.exists(KMC_TOOLS)):
        pytest.skip("oracle/_ref/kmc_ref not built")
    tmp = str(tmp_path)
    fq = os.path.join(tmp, "reads.fq")
    write_fastq_reads(fq, make_reads(7 * k + p, "short", 20000, 150, genome_len=300_000) + make_reads(p, "n_dense", 2000, 150))
    ref_db, st = count(KMC_REF, tmp, "ref", fq, k, ("-p%d" % p, "-ci2", "-sr1") + (() if both else ("-b",)))
    h, sig_map_pos, _, raw = kmc_pre_bins(ref_db + ".kmc_pre", ref_db + ".kmc_suf")
    m, sig_map = signature_map_from_kmc_pre(ref_db + ".kmc_pre")
    assert m == p and np.array_equal(sig_map, sig_map_pos)
    out = os.path.join(tmp, "gpu")
    res = count_reads([fq], out, k, m, sig_map, h["p"], h["cmin"], h["cmax"], 255, both, batch_bytes=1 << 21,
                      n_bins=raw.shape[0])
    assert md5(out + ".kmc_suf") == md5(ref_db + ".kmc_suf")
    assert md5(out + ".kmc_pre") == md5(ref_db + ".kmc_pre")
    s = st.get("Stats", st)
    assert res["n_super_kmers"] == int(s["#Total_super-k-mers"])
    assert dump_sorted(tmp, out, "gpu") == dump_sorted(tmp, ref_db, "ref")
