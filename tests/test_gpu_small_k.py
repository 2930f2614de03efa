"""Small k on the GPU (kmcb200_smallk_*, kmc_b200.SmallKCounter, kmc_b200.reads.count_reads_small_k) against the numpy model of
test_small_k_model.py, which is pinned to the reference CLI with no GPU; and, where oracle/_ref holds the reference's binaries, against
live `kmc` runs."""
import os
import subprocess
import sys

import numpy as np
import pytest

import kmc_b200
from kmc_b200 import ERR_CAPACITY, ERR_INVALID, KmcB200Error, SmallKCounter
from kmc_b200.reads import count_reads, count_reads_small_k, sequences_to_batch
from stage1_testlib import batch_of, make_reads
from test_gpu_kmc_files import KMC_REF, KMC_TOOLS, count, dump_sorted, md5, write_fastq
import test_small_k_model as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _batches():
    return {
        "short": batch_of(make_reads(1, "short", n_reads=400)),
        "long": batch_of(make_reads(2, "long", n_reads=1, read_len=5_000_000)),
        "ndense": batch_of(make_reads(3, "n_dense", n_reads=300)),
        "polya": batch_of(make_reads(4, "low_complexity", n_reads=6, read_len=3000)) + b"A" * 100_000 + b"\n",
    }


@pytest.fixture(scope="module")
def batches():
    return _batches()


@pytest.mark.parametrize("both", [True, False])
@pytest.mark.parametrize("k", list(range(1, 14)))
def test_counts_equal_the_model(batches, k, both):
    sk = SmallKCounter(k, both, max_batch_bytes=max(len(b) for b in batches.values()))
    for name, b in batches.items():
        sk.reset()
        before = sk.kernel_launches()
        sk.add(b)
        assert sk.kernel_launches() - before == 1
        got = sk.read()
        assert np.array_equal(got, M.counts(np.frombuffer(b, dtype=np.uint8), k, both)), (name, k, both)
    sk.close()


@pytest.mark.parametrize("k", [3, 7, 8, 13])
def test_several_batches_reset_and_device_twin(batches, k):
    import torch
    parts = [batches["short"], batches["ndense"], batches["polya"]]
    want = sum(M.counts(np.frombuffer(b, dtype=np.uint8), k) for b in parts)
    sk = SmallKCounter(k, max_batch_bytes=max(len(b) for b in parts))
    sk.add(b"ACGTTT\n")
    sk.reset()
    for b in parts:
        sk.add(b)
    assert np.array_equal(sk.read(), want)
    sk.reset()
    assert not sk.read().any()
    st = torch.cuda.Stream()
    dev = [torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() for b in parts]
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        for d in dev:
            sk.dev_add(d.data_ptr(), d.numel(), st.cuda_stream)
    assert np.array_equal(sk.read(), want)
    sk.close()


@pytest.mark.parametrize("k", [4, 9, 12])
def test_add_fastx_in_one_chunk_and_in_awkward_chunks(tmp_path, k):
    fq = os.path.join(str(tmp_path), "r.fq")
    write_fastq(fq, 60 + k, 600, n_frac=0.05)
    raw = open(fq, "rb").read()
    want = M.counts(sequences_to_batch(raw), k)
    px = kmc_b200.FastxParser("fastq", max_chunk_bytes=len(raw))
    sk = SmallKCounter(k, max_batch_bytes=len(raw) + 1)
    assert sk.add_fastx(px, raw) == len(raw)
    assert np.array_equal(sk.read(), want)
    sk.reset()
    pos = 0
    for cut in (1000, 1, 40_000, 333, 10 ** 9):                        # 1 byte past a record start, inside lines, then the rest
        piece = raw[pos:pos + max(cut, 2000)]
        final = pos + len(piece) >= len(raw)
        pos += sk.add_fastx(px, piece, final)
        if final:
            break
    assert pos == len(raw)
    assert np.array_equal(sk.read(), want)
    sk.close()
    px.close()


def _model_finish(b, k, both, cmin, cmax, cntmax):
    return M.finish(M.counts(np.frombuffer(b, dtype=np.uint8), k, both), k, cmin, cmax, cntmax)


@pytest.mark.parametrize("k,both,cmin,cmax,cntmax", [
    (1, True, 2, 10 ** 9, 255), (3, False, 1, 10 ** 9, 1), (5, True, 1, 1 << 33, 1 << 33), (7, True, 3, 50, 255), (8, False, 1, 10 ** 9, 1),
    (9, True, 2, 10 ** 9, 7), (11, True, 1, 10 ** 9, 65535), (12, False, 2, 3, 255), (13, True, 1, (1 << 33) + 9, 1 << 40), (13, False, 2, 10 ** 9, 255)])
def test_finish_and_emit_equal_the_model(batches, k, both, cmin, cmax, cntmax):
    b = batches["short"] + batches["polya"]
    sk = SmallKCounter(k, both, max_batch_bytes=len(b))
    sk.add(b)
    lp, cs, nbytes, stats = sk.finish(cmin, cmax, cntmax)
    e_lp, e_cs, e_recs, e_lut, e_stats = _model_finish(b, k, both, cmin, cmax, cntmax)
    assert (lp, cs, nbytes, stats) == (e_lp, e_cs, e_recs.size, e_stats)
    if nbytes:
        short = np.full(nbytes - 1, 0xAB, dtype=np.uint8)
        with pytest.raises(KmcB200Error) as ei:
            sk.emit(short)
        assert ei.value.code == ERR_CAPACITY and (short == 0xAB).all()
    recs, lut = sk.emit()
    assert np.array_equal(recs, e_recs) and np.array_equal(lut, e_lut)
    sk.add(b"ACGT\n")
    with pytest.raises(KmcB200Error) as ei:
        sk.emit()                                                       # the counts changed since finish
    assert ei.value.code == ERR_INVALID
    sk.close()


def _case_input(case, tmp):
    path = os.path.join(tmp, "input" + (".fa" if M.INPUTS[case[1]][1] == "-fa" else ".fq"))
    M.write_input(case, path)
    return path


@pytest.mark.parametrize("parse", ["host", "gpu"])
def test_databases_equal_every_stored_reference_case(tmp_path, parse):
    g = M.golden()
    for i, case in enumerate(M.CASES):
        name, _, _, k, both, cmin, cmax, cntmax = case
        tmp = str(tmp_path / name)
        os.makedirs(tmp)
        inp = _case_input(case, tmp)
        db = os.path.join(tmp, "db")
        if i % 2:
            res = count_reads_small_k([inp], db, k, cmin, cmax, cntmax, both, batch_bytes=1 << 20, parse=parse)
        else:
            res = count_reads([inp], db, k, 9, None, 7, cmin, cmax, cntmax, both, batch_bytes=1 << 20, parse=parse, small_k=True)
        ref = g[name]
        assert md5(db + ".kmc_pre") == ref["kmc_pre_md5"] and md5(db + ".kmc_suf") == ref["kmc_suf_md5"], (name, parse)
        assert (res["n_unique"], res["n_cutoff_min"], res["n_cutoff_max"], res["n_total"]) == \
            (ref["n_unique"], ref["n_cutoff_min"], ref["n_cutoff_max"], ref["n_total"])
        assert res["lut_prefix_len"] == ref["lut_prefix_len"] and res["n_super_kmers"] == 0


def test_count_reads_takes_the_small_k_path_where_bins_cannot_run_and_the_cli(tmp_path):
    case = next(c for c in M.CASES if c[0] == "k7_ci3_cx40")
    ref = M.golden()[case[0]]
    inp = _case_input(case, str(tmp_path))
    db = str(tmp_path / "db")
    count_reads([inp], db, 7, 9, None, None, 3, 40, 255)                  # k <= p, no flag
    assert md5(db + ".kmc_pre") == ref["kmc_pre_md5"] and md5(db + ".kmc_suf") == ref["kmc_suf_md5"]
    for extra in ([], ["--small-k", "-p", "5"], ["--gpu-parse"]):
        cli = str(tmp_path / ("cli%d" % len(extra)))
        subprocess.run([sys.executable, "-m", "kmc_b200.reads", "-k", "7", "--ci", "3", "--cx", "40", "--cs", "255"] + extra + [inp, cli],
                       check=True, cwd=ROOT, stdout=subprocess.DEVNULL)
        assert md5(cli + ".kmc_pre") == ref["kmc_pre_md5"] and md5(cli + ".kmc_suf") == ref["kmc_suf_md5"], extra
    # small_k=False keeps the bin path (k > p here): a KMC2 database, version word 0x200
    count_reads([inp], db, 12, 9, None, 4, 2, 255, 255, small_k=False)
    assert open(db + ".kmc_pre", "rb").read()[-12:-8] != b"\0\0\0\0"


@pytest.mark.parametrize("k", [5, 9, 11, 13])
def test_live_reference_equality(tmp_path, k):
    if not (os.path.exists(KMC_REF) and os.path.exists(KMC_TOOLS)):
        pytest.skip("oracle/_ref has no kmc_ref / kmc_tools")
    tmp = str(tmp_path)
    fq = os.path.join(tmp, "reads.fq")
    write_fastq(fq, 900 + k, 4000, n_frac=0.01)
    ref_db, st = count(KMC_REF, tmp, "ref", fq, k, ("-ci2", "-m4"))
    assert open(ref_db + ".kmc_pre", "rb").read()[-12:-8] == b"\0\0\0\0", "the reference did not take its small-k path"
    db = os.path.join(tmp, "gpu")
    res = count_reads_small_k([fq], db, k, parse="gpu")
    assert md5(db + ".kmc_pre") == md5(ref_db + ".kmc_pre") and md5(db + ".kmc_suf") == md5(ref_db + ".kmc_suf")
    assert res["n_total"] == int(st["Stats"]["#Total no. of k-mers"])
    cnt = M.counts(sequences_to_batch(open(fq, "rb").read()), k)
    exp = "".join("%s\t%d\n" % ("".join("ACGT"[(v >> (2 * (k - 1 - j))) & 3] for j in range(k)), min(int(cnt[v]), 255))
                  for v in np.flatnonzero(cnt >= 2))
    assert dump_sorted(tmp, db, "gpu") == exp


def test_invalid_parameters(batches):
    for k in (0, 14, 31):
        with pytest.raises(KmcB200Error) as ei:
            SmallKCounter(k)
        assert ei.value.code == ERR_INVALID
    sk = SmallKCounter(5, max_batch_bytes=100)
    with pytest.raises(KmcB200Error) as ei:
        sk.add(b"A" * 101)
    assert ei.value.code == ERR_INVALID
    px = kmc_b200.FastxParser("fastq", max_chunk_bytes=1000)
    with pytest.raises(KmcB200Error) as ei:
        sk.add_fastx(px, b"@r\nACGT\n+\nIIII\n" * 7)                   # bytes + 1 > max_batch_bytes
    assert ei.value.code == ERR_INVALID
    with pytest.raises(KmcB200Error) as ei:
        sk.emit()                                                       # no finish yet
    assert ei.value.code == ERR_INVALID
    with pytest.raises(KmcB200Error):
        count_reads_small_k([], "/nonexistent/x", 14)
    sk.close()
    px.close()
