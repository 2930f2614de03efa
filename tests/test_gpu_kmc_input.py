"""KMC database input on the GPU: KmcDbDecoder against the numpy model at every kind of chunk cut, on synthetic LUTs past 2^32 records
and under partial filtering; its refusals, capacity rule, device twin and launch count; the _kmcdb entry points of the splitter, the
small-k counter and the estimator against their host-batch calls; and every golden case through kmc_b200.reads on both parse paths."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from kmc_input_testlib import CASES, KMC_INPUT_GOLDEN, REFUSALS, materialize, options
from kmc_b200 import ERR_CAPACITY, ERR_INVALID, HistogramEstimator, KmcB200Error, KmcDbDecoder, SmallKCounter, Splitter
from kmc_b200.reads import (count_reads, count_reads_small_k, estimate_histogram, kmc_db_info, kmc_db_records, kmc_records_to_batch,
                            write_histogram)

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(KMC_INPUT_GOLDEN))
REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")


@pytest.fixture(scope="module")
def dbs(tmp_path_factory):
    return materialize(tmp_path_factory.mktemp("kmc_input_gpu"))


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


class _Synth:
    """A synthetic database: random records, a LUT with empty prefixes and one prefix over many tiles, first record past 2^32."""

    def __init__(self, k=31, lp=7, cs=2, n=20000, base=(1 << 32) + 11, seed=3, min_count=2, max_count=1000):
        rng = np.random.default_rng(seed)
        self.kmer_len, self.lut_prefix_len, self.counter_size = k, lp, cs
        self.suffix_bytes = (k - lp) // 4
        self.record_bytes = self.suffix_bytes + cs
        self.min_count, self.max_count = min_count, max_count
        self.total_kmers = base + n
        sizes = np.zeros(2 * 4 ** lp, dtype=np.int64)                   # two bins; most prefixes empty
        hit = rng.choice(sizes.size, min(300, sizes.size), replace=False)
        sizes[hit] = rng.integers(1, 40, hit.size)
        sizes[hit[0]] = 3000                                            # one prefix over many tiles
        sizes = sizes * n // max(1, sizes.sum())
        sizes[hit[1]] += n - sizes.sum()
        self.lut = np.concatenate([[0], base + np.cumsum(sizes)]).astype(np.uint64)
        self.lut[1:][self.lut[1:] < base] = base
        self.base = base
        self.recs = rng.integers(0, 256, (n, self.record_bytes), dtype=np.uint8)
        cnt = np.where(np.arange(n) % 2 == 0, 5, 1)                     # alternately kept and dropped
        cnt[rng.random(n) < 0.1] = 2000                                 # above max_count
        for b in range(cs):
            self.recs[:, self.suffix_bytes + b] = (cnt >> (8 * b)) & 255

    def decoder(self, max_records=1 << 16):
        return KmcDbDecoder(self.kmer_len, self.lut_prefix_len, self.counter_size, self.min_count, self.max_count, self.total_kmers, self.lut,
                            max_records=max_records)


def test_decoder_equals_model_at_every_cut():
    s = _Synth()
    dec = s.decoder()
    n = s.recs.shape[0]
    cuts = [(0, n), (0, 1), (n - 1, n), (5, 6), (100, 356), (255, 257), (0, 256), (1, 4097), (777, 19000)]
    edges = np.searchsorted(s.lut[1:], s.base + np.arange(n), side="right")
    change = np.flatnonzero(np.diff(edges)) + 1                        # prefix (and bin) boundaries
    cuts += [(int(c) - 1, int(c) + 1) for c in change[:20]] + [(int(change[0]), int(change[-1]))]
    for a, b in cuts:
        exp = kmc_records_to_batch(s, s.recs[a:b], s.base + a)
        got = dec.decode(s.recs[a:b], s.base + a)
        assert got.tobytes() == exp.tobytes(), (a, b)
        assert dec.last_kept == exp.size // (s.kmer_len + 1)
    dec.close()


@pytest.mark.parametrize("k,lp,cs", [(5, 1, 0), (10, 2, 1), (21, 5, 3), (32, 4, 1), (55, 3, 4), (128, 4, 2), (256, 4, 1)])
def test_decoder_equals_model_at_many_widths(k, lp, cs):
    s = _Synth(k=k, lp=lp, cs=cs, n=3001, base=7, seed=k)
    dec = s.decoder(4096)
    for a, b in [(0, 3001), (3, 1500), (2999, 3001)]:
        assert dec.decode(s.recs[a:b], s.base + a).tobytes() == kmc_records_to_batch(s, s.recs[a:b], s.base + a).tobytes()
    dec.close()


def test_decoder_refusals_and_capacity():
    s = _Synth(n=1000, base=0)
    for kw in ({"counter_size": 5}, {"lut_prefix_len": 6}, {"kmer_len": 0}, {"max_records": 0}):
        args = dict(kmer_len=31, lut_prefix_len=7, counter_size=2, min_count=0, max_count=10, total_kmers=1000, lut=s.lut, max_records=100)
        args.update(kw)
        with pytest.raises(KmcB200Error) as e:
            KmcDbDecoder(**args)
        assert e.value.code == ERR_INVALID
    dec = s.decoder(256)
    with pytest.raises(KmcB200Error) as e:
        dec.decode(s.recs[:257], 0)
    assert e.value.code == ERR_INVALID
    with pytest.raises(KmcB200Error) as e:
        dec.decode(s.recs[:10], 995)
    assert e.value.code == ERR_INVALID
    exp = kmc_records_to_batch(s, s.recs[:200], 0)
    out = np.zeros(exp.size - 1, dtype=np.uint8)
    with pytest.raises(KmcB200Error) as e:
        dec.decode(s.recs[:200], 0, out=out)
    assert e.value.code == ERR_CAPACITY and dec.last_seq_bytes == exp.size and not out.any()
    assert dec.decode(s.recs[:200], 0).tobytes() == exp.tobytes()
    dec.close()


def test_constant_launches_per_call():
    s = _Synth(n=60000, base=0)
    dec = s.decoder(60000)
    for n in (0, 1, 1000, 60000):
        before = dec.kernel_launches()
        dec.decode(s.recs[:n], 0)
        assert dec.kernel_launches() - before == 5
    dec.close()


def test_device_twin_on_a_busy_stream():
    import torch
    s = _Synth(n=50000)
    dec = s.decoder(50000)
    exp = kmc_records_to_batch(s, s.recs, s.base)
    st = torch.cuda.Stream()
    d_out = torch.full((exp.size + 3,), 0xAB, dtype=torch.uint8, device="cuda")
    d_res = torch.zeros(2, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)
        d_suf = torch.from_numpy(s.recs.reshape(-1).copy()).pin_memory().to("cuda", non_blocking=True)
        dec.dev_decode(d_suf.data_ptr(), s.recs.shape[0], s.base, d_out.data_ptr() + 3, exp.size, d_res.data_ptr(), st.cuda_stream)
    st.synchronize()
    res = d_res.cpu().numpy()
    out = d_out.cpu().numpy()
    assert res[0] == exp.size and res[1] == exp.size // 32 and out[3:].tobytes() == exp.tobytes() and (out[:3] == 0xAB).all()
    small = torch.zeros(exp.size - 1, dtype=torch.uint8, device="cuda")
    dec.dev_decode(d_suf.data_ptr(), s.recs.shape[0], s.base, small.data_ptr(), small.numel(), d_res.data_ptr(), None)
    torch.cuda.synchronize()
    assert d_res[0].item() == exp.size and not small.any().item()
    dec.close()


@pytest.mark.parametrize("hc", [False, True])
def test_entry_points_equal_host_batch_calls(dbs, hc):
    info = kmc_db_info(dbs["k31_cs2"])
    recs = kmc_db_records(info)
    a, b = 123, info.total_kmers - 77                                   # more than two tiles, cut inside them
    batch = kmc_records_to_batch(info, recs[a:b], a)
    dec = info.decoder(max_records=b - a)
    sig_map = np.arange((1 << 18) + 1, dtype=np.uint32) % 64
    s1, s2 = (Splitter(25, 9, sig_map, 64, max_batch_bytes=1 << 22, homopolymer_compressed=hc) for _ in range(2))
    o1, p1, f1 = s1.split_raw(batch)
    o2, p2, f2, nseq, kept = s2.split_kmcdb(dec, recs[a:b], a)
    assert nseq == batch.size and kept == batch.size // 32
    assert o1.tobytes() == o2.tobytes() and np.array_equal(p1, p2)
    assert [(f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs) for f in f1] == \
        [(f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs) for f in f2]
    k1, k2 = (SmallKCounter(11, max_batch_bytes=1 << 22, homopolymer_compressed=hc) for _ in range(2))
    k1.add(batch)
    assert k2.add_kmcdb(dec, recs[a:b], a) == kept
    assert np.array_equal(k1.read(), k2.read())
    if not hc:
        e1, e2 = (HistogramEstimator(21, 7, max_batch_bytes=1 << 22) for _ in range(2))
        e1.add(batch)
        e2.add_kmcdb(dec, recs[a:b], a)
        assert np.array_equal(e1.read(), e2.read())
        for e in (e1, e2):
            e.close()
    with pytest.raises(KmcB200Error) as e:
        Splitter(25, 9, sig_map, 64, max_batch_bytes=1 << 10).split_kmcdb(dec, recs[a:b], a)
    assert e.value.code == ERR_INVALID
    for h in (s1, s2, k1, k2, dec):
        h.close()


def _run_case(name, paths, k, opts, out, parse):
    kw = options(opts)
    if "-e" in opts:
        write_histogram(out, estimate_histogram(paths, k, parse=parse))
        return None
    common = dict(cutoff_min=kw["cutoff_min"], cutoff_max=kw["cutoff_max"], counter_max=kw["counter_max"], both_strands=kw["both_strands"],
                  parse=parse)
    if k <= 13:
        return count_reads_small_k(paths, out, k, homopolymer_compressed=kw["homopolymer_compressed"], **common)
    return count_reads(paths, out, k, kw["signature_len"], None, None, n_bins=kw["n_bins"], small_k=False, opt_out_size=kw["opt_out_size"],
                       homopolymer_compressed=kw["homopolymer_compressed"], **common)


@pytest.mark.parametrize("parse", ["host", "gpu"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_case(dbs, tmp_path, name, parse):
    inputs, k, opts = CASES[name]
    ent = GOLDEN["cases"][name]
    out = str(tmp_path / "out")
    res = _run_case(name, [dbs[i] for i in inputs], k, opts, out, parse)
    if "-e" in opts:
        assert md5(out) == ent["histogram_md5"]
        return
    assert md5(out + ".kmc_pre") == ent["kmc_pre_md5"] and md5(out + ".kmc_suf") == ent["kmc_suf_md5"]
    assert (res["n_unique"], res["n_total"]) == (ent["unique_kmers"], ent["total_kmers"])
    if k > 13:
        assert res["n_reads"] == ent["n_reads"]


@pytest.mark.parametrize("parse", ["host", "gpu"])
def test_golden_case_in_many_chunks(dbs, tmp_path, parse):
    """Chunks of 300 records: the reader thread's buffers in turn, and first_record past the first chunk."""
    inputs, k, opts = CASES["two_dbs"]
    ent = GOLDEN["cases"]["two_dbs"]
    out = str(tmp_path / "out")
    res = count_reads([dbs[i] for i in inputs], out, k, 5, None, None, cutoff_min=1, batch_bytes=300 * 32, parse=parse, small_k=False)
    assert md5(out + ".kmc_pre") == ent["kmc_pre_md5"] and md5(out + ".kmc_suf") == ent["kmc_suf_md5"]
    assert res["n_reads"] == ent["n_reads"]


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals(dbs, tmp_path, name):
    inp, k, opts, msg = REFUSALS[name]
    with pytest.raises(KmcB200Error) as e:
        _run_case(name, [dbs[inp]], k, opts, str(tmp_path / "out"), "gpu")
    assert msg in str(e.value)


def test_patched_cli_equals_reference_cli(dbs, tmp_path):
    ref, b200 = os.path.join(REF, "kmc_ref"), os.path.join(REF, "kmc_b200cli")
    if not (os.path.exists(ref) and os.path.exists(b200)):
        pytest.skip("oracle/_ref binaries not built (no reference source tree)")
    outs = []
    for binary, extra in ((ref, ["-sr1"]), (b200, [])):
        out = str(tmp_path / os.path.basename(binary))
        wd = str(tmp_path / ("wd_" + os.path.basename(binary)))
        os.makedirs(wd)
        subprocess.run([binary, "-k25", "-fkmc", "-ci1", "-p5", "-n64", "-t4", "-m2"] + extra + [dbs["k31"], out, wd], check=True, stdout=subprocess.DEVNULL,
                       env=dict(os.environ, KMC_B200_DEVICES="0", KMC_B200_SORTERS_PER_GPU="1"))
        outs.append((md5(out + ".kmc_pre"), md5(out + ".kmc_suf")))
    assert outs[0] == outs[1]
