"""GPU: homopolymer compression (`kmc -hc`) in the splitter, the signature statistics and the small-k counter, against the numpy model
(hc_testlib.homopolymer_compress fed to the uncompressed entry points and to the oracles) and against what `kmc -hc -sr1` wrote
(tests/golden/hc_reference.json)."""
import hashlib
import os

import numpy as np
import pytest

import kmc_b200
from hc_testlib import HC_CASES, PART_SYMBOLS, case_format, golden, homopolymer_compress, make_hc_reads, option, padded, write_case_input
from kmc_b200.reads import count_reads, count_reads_small_k, main as reads_main, sequences_to_batch
from stage1_testlib import Stage1Oracle, batch_of, random_map
from test_gpu_kmc_files import KMC_B200, KMC_REF, count
from test_small_k_model import counts

pytestmark = pytest.mark.gpu

BIN_CASES = [n for n, c in HC_CASES.items() if c[4] > 13 and "-e" not in c[5]]
SMALL_CASES = [n for n, c in HC_CASES.items() if c[4] <= 13]


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def split_all(sp, batch):
    out, packs, frags = sp.split_raw(batch)
    return out.tobytes(), packs.copy(), [(f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs) for f in frags]


def oracle_split(batch, k, m, sig_map, n_bins):
    e = Stage1Oracle().split(homopolymer_compress(batch).tobytes(), k, m, sig_map, n_bins)
    return e.out.tobytes(), e.pack_bytes


# ------------------------------------------------------------------------------------------------ kernel edges
def _edge_batches():
    rng = np.random.default_rng(11)
    letters = np.frombuffer(b"ACGTacgtN\n", dtype=np.uint8)
    runs = []                                                          # runs of 1..200 straddling the 64-byte spans and the 16 KiB tiles
    while sum(len(r) for r in runs) < 100_000:
        runs.append(bytes([letters[rng.integers(0, 10)]]) * int(rng.choice([1, 2, 63, 64, 65, 127, 129, int(rng.integers(1, 201))])))
    straddle = b"".join(runs)
    tile = b"C" * 16383 + b"CA" + b"a" * 62 + b"G" * 16385 + b"\n" + b"T" * 64 + b"t"
    return {
        "runs": straddle,
        "tile_seams": tile,
        "alternating_case": b"aA" * 40_000 + b"\n" + b"aCgT" * 20_000,
        "separators": b"\n" * 5000 + b"NNNN\r\r",
        "one_byte": b"G",
        "empty": b"",
        "reads": batch_of(make_hc_reads(12, "hp", 600, 400, 31)),
    }


@pytest.mark.parametrize("name", list(_edge_batches()))
def test_kernel_edges_split_and_small_k(name):
    batch = _edge_batches()[name]
    k, m, nb = 31, 9, 64
    sig_map = random_map(3, m, nb)
    sp = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=max(len(batch), 1), homopolymer_compressed=True)
    out, packs, _ = split_all(sp, batch)
    if batch:
        eo, ep = oracle_split(batch, k, m, sig_map, nb)
        assert out == eo and np.array_equal(packs, ep)
    else:
        assert out == b"" and packs.size == 0
    sp.close()
    for kk in (1, 2, 3, 4):
        sk = kmc_b200.SmallKCounter(kk, max_batch_bytes=max(len(batch), 1), homopolymer_compressed=True)
        sk.add(batch)
        assert np.array_equal(sk.read(), counts(homopolymer_compress(batch), kk)), "k = %d" % kk
        sk.close()


def test_one_base_repeated_2_pow_24_times_and_full_batches():
    n = 1 << 24
    sk = kmc_b200.SmallKCounter(2, max_batch_bytes=n, homopolymer_compressed=True)
    for batch in (b"A" * n, (b"ACGTTGCA" * (n // 8)), bytes(np.random.default_rng(1).choice(np.frombuffer(b"AACCGT\n", np.uint8), n))):
        sk.reset()
        sk.add(batch)                                                  # a batch of exactly max_batch_bytes
        assert np.array_equal(sk.read(), counts(homopolymer_compress(batch), 2))
    sk.close()
    sp = kmc_b200.Splitter(31, 9, random_map(4, 9, 32), 32, max_batch_bytes=n, homopolymer_compressed=True)
    out, _, frags = split_all(sp, b"A" * n)
    assert out == b"" and sum(f[2] for f in frags) == 0               # one base: fewer than k bases remain
    sp.close()


# ------------------------------------------------------------------------------------------------ every entry-point family
def _fastq(reads):
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)) for i, r in enumerate(reads))


def _fasta(reads):
    return b"".join(b">r%d\n" % i + b"\n".join(r[j:j + 70] for j in range(0, max(len(r), 1), 70)) + b"\n" for i, r in enumerate(reads))


def test_every_entry_point_equals_the_uncompressed_one_on_the_model():
    import torch
    reads = make_hc_reads(21, "hp", 3000, 300, 31)
    batch = batch_of(reads) + b"\n"
    model = padded(batch).tobytes()
    k, m, nb = 31, 9, 128
    sig_map = random_map(5, m, nb)
    L = len(batch) + 16
    plain = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=L)
    hc = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=L, homopolymer_compressed=True)
    want = split_all(plain, model)
    got = split_all(hc, batch)
    assert got[0] == want[0] and np.array_equal(got[1], want[1]) and got[2] == want[2]
    # device twin: the caller's batch is read and never written
    d_seq = torch.from_numpy(np.frombuffer(batch, dtype=np.uint8).copy()).cuda()
    before = d_seq.clone()
    cap = len(want[0]) + 64
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_packs = torch.zeros(len(want[1]) + 64, dtype=torch.int64, device="cuda")
    d_frags = torch.zeros(nb * 40 // 8, dtype=torch.int64, device="cuda")
    d_res = torch.zeros(5, dtype=torch.int64, device="cuda")
    hc.dev_split(d_seq.data_ptr(), len(batch), d_out.data_ptr(), cap, d_packs.data_ptr(), d_packs.numel(), d_frags.data_ptr(), d_res.data_ptr())
    torch.cuda.synchronize()
    res = d_res.cpu().numpy()
    assert res[0] == len(want[0]) and res[2] == 0 and d_out[:res[0]].cpu().numpy().tobytes() == want[0]
    assert np.array_equal(d_packs[:res[1]].cpu().numpy().view(np.uint64), want[1]) and torch.equal(d_seq, before)
    # raw chunks: FASTQ and FASTA, several chunk sizes, against the model of each chunk's batch
    for text, fmt in ((_fastq(reads), "fastq"), (_fasta(reads), "fasta")):
        for chunk in (len(text), 200_000, 65_536):
            parser = kmc_b200.FastxParser(fmt, max_chunk_bytes=chunk)
            sp = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=chunk + 1, homopolymer_compressed=True)
            ref = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=chunk + 1)
            st = kmc_b200.SignatureStats(k, m, max_batch_bytes=chunk + 1, homopolymer_compressed=True)
            st_ref = kmc_b200.SignatureStats(k, m, max_batch_bytes=chunk + 1)
            sk = kmc_b200.SmallKCounter(9, max_batch_bytes=chunk + 1, homopolymer_compressed=True)
            sk_ref = kmc_b200.SmallKCounter(9, max_batch_bytes=chunk + 1)
            pos = 0
            while pos < len(text):
                raw = text[pos:pos + chunk]
                final = pos + len(raw) == len(text)
                out, packs, frags, used, nseq = sp.split_fastx(parser, raw, final)
                seq, used2 = parser.parse(raw, final)
                assert used2 == used and nseq == seq.size                # *consumed and *seq_bytes: the parsed batch
                e_out, e_packs, e_frags = ref.split_raw(padded(seq))
                assert out.tobytes() == e_out.tobytes() and np.array_equal(packs, e_packs)
                assert [(f.n_rec, f.n_super_kmers, f.bytes) for f in frags] == [(f.n_rec, f.n_super_kmers, f.bytes) for f in e_frags]
                assert st.add_fastx(parser, raw, final) == used and sk.add_fastx(parser, raw, final) == used
                st_ref.add(padded(seq))
                sk_ref.add(padded(seq))
                pos += used
            assert np.array_equal(st.read(), st_ref.read()) and np.array_equal(sk.read(), sk_ref.read())
            for h in (parser, sp, ref, st, st_ref, sk, sk_ref):
                h.close()
    # host batch and device twin of the statistics and the small-k counter
    st, st_ref = kmc_b200.SignatureStats(k, m, max_batch_bytes=L, homopolymer_compressed=True), kmc_b200.SignatureStats(k, m, max_batch_bytes=L)
    sk, sk_ref = kmc_b200.SmallKCounter(11, max_batch_bytes=L, homopolymer_compressed=True), kmc_b200.SmallKCounter(11, max_batch_bytes=L)
    st.add(batch)
    st.dev_add(d_seq.data_ptr(), len(batch))
    sk.add(batch)
    sk.dev_add(d_seq.data_ptr(), len(batch))
    for _ in range(2):
        st_ref.add(model)
        sk_ref.add(model)
    assert np.array_equal(st.read(), st_ref.read()) and np.array_equal(sk.read(), sk_ref.read()) and torch.equal(d_seq, before)
    for h in (plain, hc, st, st_ref, sk, sk_ref):
        h.close()


def test_off_means_off_and_three_launches_per_call():
    batch = batch_of(make_hc_reads(31, "hp", 500, 300, 31))
    k, m, nb = 31, 9, 32
    sig_map = random_map(6, m, nb)
    never = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=len(batch))
    toggled = kmc_b200.Splitter(k, m, sig_map, nb, max_batch_bytes=len(batch))
    toggled.set_homopolymer_compressed(True)
    on = split_all(toggled, batch)                                     # sizes the output buffers (split_raw may call twice)
    a0 = toggled.kernel_launches()
    assert split_all(toggled, batch)[0] == on[0]
    on_launches = toggled.kernel_launches() - a0
    toggled.set_homopolymer_compressed(False)
    split_all(never, batch)
    split_all(toggled, batch)
    b0, c0 = never.kernel_launches(), toggled.kernel_launches()
    r_never, r_off = split_all(never, batch), split_all(toggled, batch)
    off_launches, never_launches = toggled.kernel_launches() - c0, never.kernel_launches() - b0
    assert r_off[0] == r_never[0] and np.array_equal(r_off[1], r_never[1]) and r_off[2] == r_never[2]
    assert off_launches == never_launches and on_launches == never_launches + 3
    assert on[0] != r_never[0]
    for cls, args in ((kmc_b200.SignatureStats, (k, m)), (kmc_b200.SmallKCounter, (7,))):
        n, t = cls(*args, max_batch_bytes=len(batch)), cls(*args, max_batch_bytes=len(batch))
        t.set_homopolymer_compressed(True)
        t.add(batch)
        assert t.kernel_launches() == 1 + 3
        t.reset()
        t.set_homopolymer_compressed(False)
        l_n, l_t = n.kernel_launches(), t.kernel_launches()
        n.add(batch)
        t.add(batch)
        assert np.array_equal(n.read(), t.read()) and n.kernel_launches() - l_n == t.kernel_launches() - l_t == 1
        n.close()
        t.close()
    never.close()
    toggled.close()


# ------------------------------------------------------------------------------------------------ against kmc -hc
def _input(tmp_path, case):
    path = os.path.join(str(tmp_path), case + ".input")
    write_case_input(case, path)
    assert md5(path) == golden()[case]["input_md5"]
    return path


@pytest.mark.parametrize("parse", ["host", "gpu"])
@pytest.mark.parametrize("case", BIN_CASES + SMALL_CASES)
def test_count_reads_equals_kmc_hc(tmp_path, case, parse):
    c = golden()[case]
    seed, profile, n_reads, read_len, k, opts = HC_CASES[case]
    path = _input(tmp_path, case)
    out = os.path.join(str(tmp_path), "db")
    cmin, cmax, cs = option(case, "-ci", 2), option(case, "-cx", 1_000_000_000), option(case, "-cs", 255)
    both = "-b" not in opts
    if k <= 13:
        res = count_reads_small_k([path], out, k, cmin, cmax, cs, both, batch_bytes=1 << 22, parse=parse, homopolymer_compressed=True)
    else:
        res = count_reads([path], out, k, option(case, "-p", 9), None, None, cmin, cmax, cs, both, batch_bytes=1 << 22, n_bins=option(case, "-n", 512),
                          parse=parse, opt_out_size="--opt-out-size" in opts, homopolymer_compressed=True)
        assert res["n_super_kmers"] == c["total_super_kmers"] and res["lut_prefix_len"] == c["header"]["p"]
        assert res["n_reads"] == n_reads and res["n_bases"] == sequences_to_batch(open(path, "rb").read()).size
    assert res["n_kmers"] == c["total_kmers"] and res["n_unique"] == c["unique_kmers"]
    assert md5(out + ".kmc_pre") == c["kmc_pre_md5"] and md5(out + ".kmc_suf") == c["kmc_suf_md5"]
    if os.path.exists(KMC_REF) and parse == "host":                    # the live reference, where it was built
        db, _ = count(KMC_REF, str(tmp_path), "ref", path, k, tuple(o for o in opts if o not in ("-fa", "-fm")) + ("-hc", "-sr1"), fmt=case_format(case))
        assert md5(db + ".kmc_pre") == md5(out + ".kmc_pre") and md5(db + ".kmc_suf") == md5(out + ".kmc_suf")


def test_cli_hc_and_e_hc(tmp_path):
    """`--hc` on the command line; `-e --hc` writes the file `kmc -e -hc` (= `kmc -e`) writes."""
    case = "k31_p9_opt"
    path = _input(tmp_path, case)
    out = os.path.join(str(tmp_path), "cli")
    assert reads_main(["--hc", "-k31", "-p9", "-n64", "--ci", "1", "--opt-out-size", "--gpu-parse", "--batch-bytes", str(1 << 22), path, out]) == 0
    assert md5(out + ".kmc_pre") == golden()[case]["kmc_pre_md5"] and md5(out + ".kmc_suf") == golden()[case]["kmc_suf_md5"]
    path = _input(tmp_path, "k31_e")
    hist = os.path.join(str(tmp_path), "hist.txt")
    assert reads_main(["-e", "--hc", "-k31", path, hist]) == 0
    assert md5(hist) == golden()["k31_e"]["histogram_md5"]


@pytest.mark.parametrize("k", [31, 55])
def test_patched_binary_equals_kmc_hc(tmp_path, k):
    """kmc_b200cli -hc: the reference's own stage 1 compresses, the GPU stage 2 counts its bins."""
    for b in (KMC_REF, KMC_B200):
        if not os.path.exists(b):
            pytest.skip("%s not built" % os.path.basename(b))
    case = "k31_p9" if k == 31 else "k55_p11"
    path = _input(tmp_path, case)
    opts = tuple(HC_CASES[case][5]) + ("-hc",)
    ref_db, _ = count(KMC_REF, str(tmp_path), "ref", path, k, opts + ("-sr1",))
    gpu_db, _ = count(KMC_B200, str(tmp_path), "gpu", path, k, opts, env={"KMC_B200_DEVICES": "0", "KMC_B200_SORTERS_PER_GPU": "1"})
    assert md5(gpu_db + ".kmc_pre") == md5(ref_db + ".kmc_pre") and md5(gpu_db + ".kmc_suf") == md5(ref_db + ".kmc_suf")


def test_long_records_match_the_model(tmp_path):
    """Records longer than the reference's part length (524,296 symbols): the GPU compresses each whole, so the database is the one of the
    reads compressed whole, counted without compression.  They are not compared with kmc_ref, which compresses each part on its own."""
    short = make_hc_reads(41, "hp", 24_000, 300, 31)
    reads = [b"".join(short[i::4]) for i in range(4)]                  # homopolymer-rich records of about 0.9 M symbols
    assert min(len(r) for r in reads) > PART_SYMBOLS
    tmp = str(tmp_path)
    raw, pre = os.path.join(tmp, "raw.fq"), os.path.join(tmp, "pre.fq")
    open(raw, "wb").write(_fastq(reads))
    open(pre, "wb").write(_fastq([homopolymer_compress(r).tobytes() for r in reads]))
    for parse in ("host", "gpu"):
        a = count_reads([raw], os.path.join(tmp, "a"), 31, 9, None, 7, 1, parse=parse, batch_bytes=1 << 24, n_bins=64, homopolymer_compressed=True)
        b = count_reads([pre], os.path.join(tmp, "b"), 31, 9, None, 7, 1, parse=parse, batch_bytes=1 << 24, n_bins=64)
        assert (a["n_kmers"], a["n_unique"], a["n_super_kmers"]) == (b["n_kmers"], b["n_unique"], b["n_super_kmers"])
        for ext in (".kmc_pre", ".kmc_suf"):
            assert md5(os.path.join(tmp, "a") + ext) == md5(os.path.join(tmp, "b") + ext)
        sa = count_reads_small_k([raw], os.path.join(tmp, "sa"), 9, 1, parse=parse, batch_bytes=1 << 24, homopolymer_compressed=True)
        sb = count_reads_small_k([pre], os.path.join(tmp, "sb"), 9, 1, parse=parse, batch_bytes=1 << 24)
        assert sa["n_total"] == sb["n_total"] and md5(os.path.join(tmp, "sa.kmc_suf")) == md5(os.path.join(tmp, "sb.kmc_suf"))
