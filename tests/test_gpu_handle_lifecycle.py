"""Destroy gives back what create and use took: for each of the five device handles, the free memory of the GPU after
create -> one small input (so that the buffers grown on demand exist) -> destroy is what it was before.  The first cycle of a handle is
not measured: it loads the library's kernels and warms the runtime, which stays.  Other processes may share the GPU, so a handle's
leak is told from their traffic by size: every cycle here allocates tens of MiB, the tolerance is a few."""
import numpy as np
import pytest

from kmc_testlib import bin_extras, fast_bin

pytestmark = pytest.mark.gpu

TOLERANCE = 8 << 20          # allocator granularity (2 MiB blocks) and neighbours on a shared GPU


def _free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def _returns_memory(cycle):
    cycle()                       # not measured: module load, first-use allocations of the runtime
    before = _free_bytes()
    used = cycle()
    after = _free_bytes()
    assert used > 2 * TOLERANCE, "the cycle allocated too little (%d bytes) for a leak to show" % used
    assert before - after <= TOLERANCE, "%d bytes of device memory were not given back" % (before - after)


@pytest.fixture(scope="module")
def reads_batch():
    from stage1_testlib import batch_of, make_reads
    return batch_of(make_reads(11, "short", n_reads=3000))


@pytest.fixture(scope="module")
def fastq_chunk():
    from test_fastx_model import fastq_text
    return fastq_text(2026, 2000, max_len=200)


def test_stage2_context_returns_its_memory(monkeypatch):
    """One ordinary bin, one indexed bin and one bin counted key block by key block, over two slots."""
    import kmc_b200
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", "150000")
    small, big = fast_bin(41, 31, 120_000), fast_bin(42, 31, 2_000_000)
    extras, psk = bin_extras(small)

    def cycle():
        start = _free_bytes()
        ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(31, True, 2, 10 ** 9, 255, 7), device=0, n_slots=2)
        skb = kmc_b200.SuperKmerBin(data=small.data, n_rec=small.n_rec, pack_bytes=small.pack_bytes, kmer_len=31)
        ctx.process_bin(skb)
        data = np.ascontiguousarray(small.data)
        packs = np.ascontiguousarray(small.pack_bytes, dtype=np.uint64)
        out = np.zeros(ctx.out_capacity(small.n_rec) + 64, dtype=np.uint8)
        lut = np.zeros(ctx.lut_entries, dtype=np.uint64)
        ctx.submit_bin_indexed(1, data.ctypes.data, data.size, small.n_rec, packs, extras, psk, out.ctypes.data, out.size, lut.ctypes.data)
        ctx.wait_bin(1)
        launches = ctx.kernel_launches()
        ctx.process_bin(kmc_b200.SuperKmerBin(data=big.data, n_rec=big.n_rec, pack_bytes=big.pack_bytes, kmer_len=31))
        assert ctx.kernel_launches() - launches > 40, "the big bin was not counted in key blocks"
        used = start - _free_bytes()
        ctx.close()
        return used

    _returns_memory(cycle)


def test_splitter_returns_its_memory(reads_batch):
    import kmc_b200
    from stage1_testlib import random_map
    sig_map = random_map(7, 9, 64)

    def cycle():
        start = _free_bytes()
        sp = kmc_b200.Splitter(31, 9, sig_map, 64, max_batch_bytes=1 << 22)
        sp.count_kxmers()
        out, packs, frags = sp.split_raw(reads_batch)
        assert out.size and sp.kernel_launches() >= 10
        used = start - _free_bytes()
        sp.close()
        return used

    _returns_memory(cycle)


def test_signature_stats_return_their_memory(reads_batch):
    import kmc_b200

    def cycle():
        start = _free_bytes()
        st = kmc_b200.SignatureStats(31, 9, max_batch_bytes=1 << 26)
        st.add(reads_batch)
        assert int(st.read().sum()) > 0
        used = start - _free_bytes()
        st.close()
        return used

    _returns_memory(cycle)


def test_fastx_parser_returns_its_memory(fastq_chunk):
    import kmc_b200

    def cycle():
        start = _free_bytes()
        fx = kmc_b200.FastxParser(kmc_b200.FASTQ, max_chunk_bytes=1 << 25)
        seq, used_bytes = fx.parse(fastq_chunk)
        assert used_bytes == len(fastq_chunk) and seq.size
        used = start - _free_bytes()
        fx.close()
        return used

    _returns_memory(cycle)


def test_small_k_counter_returns_its_memory(reads_batch, tmp_path):
    """k = 12: 4^12 counters; write_db grows the record and LUT buffers of the emit."""
    import kmc_b200

    def cycle():
        start = _free_bytes()
        sk = kmc_b200.SmallKCounter(12, max_batch_bytes=1 << 25)
        sk.add(reads_batch)
        totals = sk.write_db(str(tmp_path / "small_k"), cutoff_min=1)
        assert totals[0] > 0
        used = start - _free_bytes()
        sk.close()
        return used

    _returns_memory(cycle)
