"""GPU: the library driven as KMC drives it.  Several stage-2 contexts on one device, each on its own host thread (the KMC shim's
sorter threads); every handle kind at once; thread-local create errors; the device entry points on a caller stream that is still busy;
and the ordering rule of include/kmc_b200.h between device-form and host-form calls on one handle or slot.  Inputs and expected results
are built in the main thread before any thread starts; every result is compared with an oracle and, where the handle has state, with
the same handle's result when it runs alone."""
import ctypes as C
import gc
import os
import threading
import time

import numpy as np
import pytest

import kmc_b200
from kmc_b200 import KmcB200Error, Stage2Context, Stage2Params
from kmc_b200.reads import count_reads, count_reads_small_k, sequences_to_batch
from kmc_testlib import Params, bin_from_reads, choose_lut_prefix_len, fast_bin, synth_bin, to_skb
from stage0_testlib import oracle_signature_stats
from stage1_testlib import Stage1Oracle, batch_of, make_reads, random_map
from gzip_testlib import bgzf, inflate_all
from test_db_writer import parse_db
from test_fastx_model import fastq_text
from test_gpu_kmc_files import write_fastq
import estimate_testlib as et
import test_small_k_model as M

pytestmark = pytest.mark.gpu

SLEEP_MS = 50                       # how long _busy keeps the caller's stream asleep before the input copy
KB_LIMIT = 1 << 19                  # KMCB200_MAX_BLOCK_RECORDS of the key-block context: the 1.3e6 k-mer bin is counted in several blocks
KB_CHUNK = 1 << 18                  # KMCB200_MAX_CHUNK_BYTES: ... and expanded in chunks


def run_together(fns):
    """Runs every fn on its own thread, all released by one barrier; returns their results, raises the first failure."""
    barrier = threading.Barrier(len(fns))
    res, err = [None] * len(fns), [None] * len(fns)

    def body(i):
        try:
            barrier.wait()
            res[i] = fns[i]()
        except BaseException as e:              # noqa: B902 - re-raised in the main thread
            err[i] = e
            barrier.abort()

    ts = [threading.Thread(target=body, args=(i,)) for i in range(len(fns))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    real = [e for e in err if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if real or any(err):
        raise (real or [e for e in err if e is not None])[0]
    return res


def s2params(p):
    return Stage2Params(p.k, p.both_strands, p.cutoff_min, p.cutoff_max, p.counter_max, p.lut_prefix_len)


def same(got, want, what):
    """A stage-2 result (payload bytes, raw LUT, stats) byte-equal to the oracle's."""
    payload, lut, stats = got
    assert stats == tuple(want.stats), what
    assert payload == want.payload, what
    assert np.array_equal(lut, want.lut), what


def host_result(r):
    return r.payload.tobytes(), r.lut.copy(), r.stats


# ---------------------------------------------------------------------------------------------------------------------- inputs
_cache = {}


def _bins_for(k, big):
    """sizes 0, 1, ~2e4, ~3e5 k-mers (and ~1.3e6 for the key-block context), seeded by k."""
    key = (k, big)
    if key not in _cache:
        bins = [synth_bin(0, k, 0), bin_from_reads(k, ["ACGTTGCAAGGCTTACCGATGCATGCAATCGGATCCTAGGCTAACGTACGATCGATGCATCGATGCATCGATGCATCGATCGAAGCTGCATGCAGTCCAGTGACGTACGTAGCTAGCTAGCATCGATCGACTGACTGCATGCA"[:k]]),
                synth_bin(10 + k, k, 1700, genome_len=6000), fast_bin(20 + k, k, 300_000)]
        if big:
            bins.append(fast_bin(30 + k, k, 1_300_000))
        _cache[key] = bins
    return _cache[key]


def _params(k, both):
    return Params(k=k, both_strands=both, lut_prefix_len=choose_lut_prefix_len(k))


def _expected(oracle, k, both, big):
    key = ("e", k, both, big)
    if key not in _cache:
        p = _params(k, both)
        _cache[key] = [oracle.process_bin(b, p) for b in _bins_for(k, big)]
    return _cache[key]


# ---------------------------------------------------------------------------------------------------------------------- the GIL
def test_library_calls_release_the_gil():
    """kmc_b200 binds the library with ctypes.CDLL, which drops the GIL for the length of every call: another Python thread runs at full
    speed while one call (a 1 GiB device-to-host copy of the estimator's counters) is inside the library.  Without that the threads of
    the tests below would take turns instead of overlapping."""
    assert type(kmc_b200.load_library()) is C.CDLL
    batch = batch_of(make_reads(7, "short", n_reads=50))
    est = kmc_b200.HistogramEstimator(31, max_batch_bytes=len(batch))
    est.add(batch)
    ticks, stop = [0], threading.Event()

    def spin():
        while not stop.is_set():
            ticks[0] += 1

    t = threading.Thread(target=spin)
    t.start()
    try:
        time.sleep(0.05)
        t0, n0 = time.perf_counter(), ticks[0]
        time.sleep(0.05)                    # (time.sleep drops the GIL: the spinner's full rate)
        rate = (ticks[0] - n0) / (time.perf_counter() - t0)
        t0, n0 = time.perf_counter(), ticks[0]
        counters = est.read()
        dt, dn = time.perf_counter() - t0, ticks[0] - n0
    finally:
        stop.set()
        t.join()
        est.close()
    assert _sparse(et.SparseCounters.from_dense(counters.reshape(-1))) == _sparse(et.SparseCounters(et.oracle_increments(batch, 31, 7)))
    assert dt > 0.03, dt                    # long against the interpreter's 5 ms switch interval
    assert dn > 0.3 * rate * dt, (dn, rate, dt)


# ---------------------------------------------------------------------------------------------------------------------- part 1
# (k, canonical) of each thread's context; thread 0's context counts the 1.3e6 k-mer bin in key blocks, thread 1 uses the device form
THREADS = {2: [(31, True), (55, False)], 3: [(31, True), (128, False), (55, True)], 4: [(31, True), (55, False), (128, True), (31, False)]}
PARALLEL_CASES = [(2, 1, False), (2, 2, False), (3, 1, True), (4, 1, False)]


def _host_thread(ctx, bins, slots):
    """The thread's bins twice through the host form: process_bin, or submit/wait over two slots (bin i+1 in flight while i is waited)."""
    out = []
    seq = list(bins) * 2
    if slots == 1:
        return [host_result(ctx.process_bin(to_skb(b))) for b in seq]
    datas = [np.ascontiguousarray(b.data) for b in seq]
    caps = [ctx.out_capacity(b.n_rec) + 64 for b in seq]
    outs = [np.zeros(c, dtype=np.uint8) for c in caps]
    luts = [np.zeros(ctx.lut_entries, dtype=np.uint64) for _ in seq]
    packs = [np.ascontiguousarray(b.pack_bytes, dtype=np.uint64) for b in seq]

    def submit(i):
        ctx.submit_bin(i % 2, datas[i].ctypes.data, datas[i].size, seq[i].n_rec, packs[i], outs[i].ctypes.data, caps[i], luts[i].ctypes.data)

    submit(0)
    for i in range(len(seq)):
        if i + 1 < len(seq):
            submit(i + 1)
        nbytes, stats = ctx.wait_bin(i % 2)
        out.append((outs[i][:nbytes].tobytes(), luts[i], stats))
    return out


def _dev_buffers(ctx, bins):
    import torch
    seq = list(bins) * 2
    bufs = []
    for b in seq:
        d_bin = torch.zeros(b.size + 64, dtype=torch.uint8, device="cuda")
        if b.size:
            d_bin[:b.size] = torch.from_numpy(np.ascontiguousarray(b.data))
        cap = ctx.out_capacity(b.n_rec) + 64
        bufs.append((b, d_bin, torch.zeros(cap, dtype=torch.uint8, device="cuda"), cap, torch.zeros(ctx.lut_entries, dtype=torch.int64, device="cuda"),
                     torch.zeros(8, dtype=torch.int64, device="cuda")))
    torch.cuda.synchronize()
    return bufs


def _run_dev(ctx, bufs, stream):
    for b, d_bin, d_out, cap, d_lut, d_res in bufs:
        ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), stream.cuda_stream)
    stream.synchronize()
    out = []
    for b, d_bin, d_out, cap, d_lut, d_res in bufs:
        r = d_res.cpu().numpy().view(np.uint64)
        assert int(r[5]) == 0 and int(r[6]) == 0, r
        out.append((d_out[:int(r[4]) * ctx.out_rec_bytes].cpu().numpy().tobytes(), d_lut.cpu().numpy().view(np.uint64), tuple(int(x) for x in r[:4])))
    return out


def _db_thread(ctx, w, bins):
    """test_db_writer.test_gpu_bins_straight_into_the_database on one thread: the bins twice, straight into the thread's own database."""
    seq = list(bins) * 2
    lut = np.zeros(ctx.lut_entries, dtype=np.uint64)
    for i, b in enumerate(seq):
        data = np.ascontiguousarray(b.data)
        cap = ctx.out_capacity(b.n_rec) + 64
        ptr = w.reserve(cap)
        ctx.submit_bin(0, data.ctypes.data, data.size, b.n_rec, np.ascontiguousarray(b.pack_bytes, dtype=np.uint64), ptr, cap, lut.ctypes.data)
        nbytes, stats = ctx.wait_bin_scanned(0, w.records)
        w.commit_bin(nbytes, lut, stats, [i])
    return w.close()


@pytest.mark.parametrize("n_threads,n_slots,with_db", PARALLEL_CASES, ids=["%dthreads-%dslots%s" % (n, s, "-db" if d else "") for n, s, d in PARALLEL_CASES])
def test_parallel_contexts_on_one_device(oracle, monkeypatch, tmp_path, n_threads, n_slots, with_db):
    """One context per thread on device 0, all counting at once; every payload, LUT and stats tuple byte-equal to the oracle's."""
    import torch
    cfg = THREADS[n_threads]
    bins = [_bins_for(k, i == 0) for i, (k, both) in enumerate(cfg)]
    want = [_expected(oracle, k, both, i == 0) for i, (k, both) in enumerate(cfg)]
    monkeypatch.setenv("KMCB200_MAX_BLOCK_RECORDS", str(KB_LIMIT))
    monkeypatch.setenv("KMCB200_MAX_CHUNK_BYTES", str(KB_CHUNK))
    ctxs = [Stage2Context(s2params(_params(*cfg[0])), device=0, n_slots=n_slots)]
    monkeypatch.delenv("KMCB200_MAX_BLOCK_RECORDS")
    monkeypatch.delenv("KMCB200_MAX_CHUNK_BYTES")
    ctxs += [Stage2Context(s2params(_params(k, both)), device=0, n_slots=n_slots) for k, both in cfg[1:]]
    try:
        if with_db:
            writers = []
            for i, (k, both) in enumerate(cfg):
                p = _params(k, both)
                writers.append(kmc_b200.DbWriter(os.path.join(str(tmp_path), "db%d" % i), k, p.counter_bytes, p.lut_prefix_len, 9, p.cutoff_min,
                                                 p.cutoff_max, both, staging_bytes=1 << 24))
            totals = run_together([lambda i=i: _db_thread(ctxs[i], writers[i], bins[i]) for i in range(n_threads)])
            for i, (k, both) in enumerate(cfg):
                exp = want[i] * 2
                assert totals[i] == tuple(sum(e.stats[j] for e in exp) for j in range(4)), i
                d = parse_db(os.path.join(str(tmp_path), "db%d" % i))
                assert (d["k"], d["p"], d["both"]) == (k, _params(k, both).lut_prefix_len, both)
                ends = np.append(d["luts"][1:, 0], np.uint64(d["n_recs"]))
                for j, e in enumerate(exp):
                    raw = np.diff(np.append(d["luts"][j], ends[j]).astype(np.int64)).astype(np.uint64)
                    assert d["payloads"][j] == e.payload and np.array_equal(raw, e.lut), (i, j)
            return
        stream = torch.cuda.Stream()
        bufs = _dev_buffers(ctxs[1], bins[1])
        fns = [lambda i=i: _host_thread(ctxs[i], bins[i], n_slots) for i in range(n_threads)]
        fns[1] = lambda: _run_dev(ctxs[1], bufs, stream)
        got = run_together(fns)
        for i in range(n_threads):
            exp = want[i] * 2
            assert len(got[i]) == len(exp)
            for j, (g, e) in enumerate(zip(got[i], exp)):
                same(g, e, "thread %d (k=%d, %s), bin %d" % (i, cfg[i][0], "canonical" if cfg[i][1] else "-b", j))
    finally:
        for c in ctxs:
            c.close()


# ---------------------------------------------------------------------------------------------------------------------- part 2
def _batches(seed, n=4):
    return [batch_of(make_reads(seed + i, prof, n_reads=120, read_len=200)) for i, prof in enumerate(["short", "n_dense", "short", "low_complexity"][:n])]


def _split_loop(sp, batches):
    out = []
    for b in batches:
        o, pk, fr = sp.split_raw(b)
        out.append((o.tobytes(), pk.copy(), [(f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs) for f in fr]))
    return out, sp.kxmer_totals()


def _gunzip_loop(gz, raws):
    out = []
    for raw in raws:
        text = np.zeros(1 << 20, dtype=np.uint8)
        pos, pieces = 0, []
        while pos < len(raw):
            used, n = gz.inflate(raw[pos:pos + gz.max_in_bytes], text)
            assert used, pos
            pieces.append(text[:n].tobytes())
            pos += used
        out.append(b"".join(pieces))
    return out


def test_every_handle_kind_at_once(oracle):
    """One thread per handle kind on one device, each over several batches: every result equals the same handle's result alone and the
    handle's oracle."""
    s1 = Stage1Oracle()
    K, SIG, NB = 31, 9, 64
    batches = _batches(100)
    sig_map = random_map(5, SIG, NB)
    fq = [fastq_text(200 + i, 300) for i in range(4)]
    texts = [b"".join(fq[i:i + 2]) * 4 for i in range(3)]
    raws = [bgzf(t, seed=i) for i, t in enumerate(texts)]
    p2 = _params(31, True)
    s2bins = _bins_for(31, False)[1:]
    mx = max(len(b) for b in batches)

    def make():
        sp = kmc_b200.Splitter(K, SIG, sig_map, n_bins=NB, max_batch_bytes=mx)
        sp.count_kxmers(True)
        return dict(split=sp, sig=kmc_b200.SignatureStats(K, SIG, max_batch_bytes=mx), sk7=kmc_b200.SmallKCounter(7, max_batch_bytes=mx),
                    sk12=kmc_b200.SmallKCounter(12, False, max_batch_bytes=mx), est=kmc_b200.HistogramEstimator(K, max_batch_bytes=mx),
                    fx=kmc_b200.FastxParser("fastq", max_chunk_bytes=max(len(f) for f in fq)), gz=kmc_b200.Gunzip(0, 1 << 22, 1 << 20),
                    s2=Stage2Context(s2params(p2)))

    def work(h):
        def adds(name):
            for b in batches:
                h[name].add(b)
            return h[name].read()
        return dict(split=lambda: _split_loop(h["split"], batches), sig=lambda: adds("sig"), sk7=lambda: adds("sk7"), sk12=lambda: adds("sk12"),
                    est=lambda: (_sparse(et.SparseCounters.from_dense(adds("est").reshape(-1))), h["est"].histogram()), fx=lambda: [h["fx"].parse(f)[0].tobytes() for f in fq],
                    gz=lambda: _gunzip_loop(h["gz"], raws), s2=lambda: [host_result(h["s2"].process_bin(to_skb(b))) for b in s2bins])

    def close(h):
        for x in h.values():
            x.close()

    alone_h = make()
    try:
        alone = {name: fn() for name, fn in work(alone_h).items()}
    finally:
        close(alone_h)
    h = make()
    try:
        names = list(work(h))
        got = dict(zip(names, run_together([work(h)[n] for n in names])))
    finally:
        close(h)
    # the single-threaded run of the same handles
    for name in ("sig", "sk7", "sk12"):
        assert np.array_equal(got[name], alone[name]), name
    assert got["fx"] == alone["fx"] and got["gz"] == alone["gz"]
    assert got["est"][0] == alone["est"][0] and np.array_equal(got["est"][1], alone["est"][1])
    assert np.array_equal(got["split"][1], alone["split"][1])
    for (o, pk, fr), (o2, pk2, fr2) in zip(got["split"][0], alone["split"][0]):
        assert o == o2 and np.array_equal(pk, pk2) and fr == fr2
    # the oracles
    for (o, pk, fr), b in zip(got["split"][0], batches):
        want = s1.split(b, K, SIG, sig_map, NB)
        assert o == want.out.tobytes() and np.array_equal(pk, want.pack_bytes)
        assert np.array_equal(np.array(fr, dtype=np.uint64), want.frags)
    assert np.array_equal(got["sig"], sum(oracle_signature_stats(b, K, SIG).astype(np.uint64) for b in batches).astype(np.uint32))
    assert np.array_equal(got["sk7"], sum(M.counts(np.frombuffer(b, np.uint8), 7) for b in batches))
    assert np.array_equal(got["sk12"], sum(M.counts(np.frombuffer(b, np.uint8), 12, False) for b in batches))
    assert got["est"][0] == _sparse(et.SparseCounters(np.concatenate([et.oracle_increments(b, K, 7) for b in batches])))
    assert np.array_equal(got["est"][1], et.oracle_histogram(b"\n".join(batches), K, 7))
    assert got["fx"] == [sequences_to_batch(f).tobytes() for f in fq]
    assert got["gz"] == [inflate_all(r) for r in raws] == texts
    for g, e in zip(got["s2"], _expected(oracle, 31, True, False)[1:]):
        same(g, e, "stage 2 next to the other handles")


def test_count_reads_next_to_count_reads_small_k(tmp_path):
    """count_reads(parse="gpu") (its reader thread, the writer's thread, stage 0 and the split) on one thread and count_reads_small_k on
    another: the same .kmc_pre / .kmc_suf as the same calls one after the other."""
    t = str(tmp_path)
    fq = os.path.join(t, "r.fq")
    write_fastq(fq, 11, 6000)
    calls = [lambda tag: count_reads([fq], os.path.join(t, tag + "_big"), 31, 9, None, batch_bytes=1 << 18, parse="gpu"),
             lambda tag: count_reads_small_k([fq], os.path.join(t, tag + "_small"), 9, batch_bytes=1 << 18, parse="gpu")]
    for c in calls:
        c("seq")
    run_together([lambda c=c: c("par") for c in calls])
    for name in ("big", "small"):
        for ext in (".kmc_pre", ".kmc_suf"):
            a = open(os.path.join(t, "seq_" + name + ext), "rb").read()
            b = open(os.path.join(t, "par_" + name + ext), "rb").read()
            assert a == b, name + ext


# ---------------------------------------------------------------------------------------------------------------------- part 3
def _failing_creates():
    """(create that fails, the words its message must hold, family of the last_error symbol)"""
    return [
        (lambda: Stage2Context(Stage2Params(0, True, 2, 10 ** 9, 255, 7)), "kmer_len 0", "kmcb200"),
        (lambda: kmc_b200.Splitter(31, 4, np.zeros(257, np.uint32)), "signature_len 4", "kmcb200_splitter"),
        (lambda: kmc_b200.SignatureStats(31, 12), "signature_len 12", "kmcb200_sigstats"),
        (lambda: kmc_b200.SmallKCounter(14), "kmer_len 14", "kmcb200_smallk"),
        (lambda: kmc_b200.HistogramEstimator(31, s=8), "s 8", "kmcb200_estimator"),
        (lambda: kmc_b200.FastxParser(3), "format 3", "kmcb200_fastx"),
        (lambda: kmc_b200.Gunzip(0, 0, 1 << 16), "max_in_bytes 0", "kmcb200_gunzip"),
    ]


FAMILIES = ["kmcb200", "kmcb200_splitter", "kmcb200_sigstats", "kmcb200_smallk", "kmcb200_estimator", "kmcb200_fastx", "kmcb200_gunzip"]


def _valid_round(sig_map):
    for h in (Stage2Context(Stage2Params(31, True, 2, 10 ** 9, 255, 7)), kmc_b200.Splitter(31, 5, sig_map, max_batch_bytes=1 << 16),
              kmc_b200.SignatureStats(31, 5, max_batch_bytes=1 << 16), kmc_b200.SmallKCounter(5, max_batch_bytes=1 << 16),
              kmc_b200.FastxParser("fasta", max_chunk_bytes=1 << 16), kmc_b200.Gunzip(0, 1 << 16, 1 << 16)):
        h.close()


def test_create_errors_are_per_thread():
    """Thread A keeps failing every create and reads its own message from last_error(NULL); thread B keeps creating and destroying valid
    handles and its last_error(NULL) stays empty.  Device memory is back where it started afterwards.  Every failing create here is
    refused while its parameters are checked, before it allocates, so the memory check covers thread B's create / destroy rounds; the
    clean-up of a create that fails after allocating (create_failed) would need an allocation to fail, and is not exercised."""
    import torch
    lib = kmc_b200.load_library()
    sig_map = np.zeros((1 << 10) + 1, np.uint32)
    _valid_round(sig_map)                               # modules loaded, first allocations made: what stays is the baseline
    for make, _, _ in _failing_creates():
        with pytest.raises(KmcB200Error):
            make()
    rounds = 40

    def a():
        for _ in range(rounds):
            for make, words, fam in _failing_creates():
                with pytest.raises(KmcB200Error) as e:
                    make()
                assert words in str(e.value), (fam, str(e.value))
                msg = getattr(lib, fam + "_last_error")(None).decode()
                assert words in msg and msg in str(e.value), (fam, msg)

    def b():
        for _ in range(rounds // 4):
            _valid_round(sig_map)
            for fam in FAMILIES:
                assert getattr(lib, fam + "_last_error")(None) == b"", fam

    # The device is shared: another process may allocate between the two readings.  A leak of ours shows in every attempt.
    for _ in range(3):
        gc.collect()
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        run_together([a, b])
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info(0)[0]
        if free1 >= free0 - (8 << 20):
            break
    assert free1 >= free0 - (8 << 20), (free0, free1)


# ---------------------------------------------------------------------------------------------------------------------- parts 4, 5
_sleep_cycles = []


def sleep_cycles():
    """The torch.cuda._sleep argument that keeps a stream busy for SLEEP_MS on this device, from one timed sleep (CUDA events)."""
    import torch
    if not _sleep_cycles:
        n = 20_000_000
        torch.cuda._sleep(n)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.cuda._sleep(n)
        e1.record()
        e1.synchronize()
        _sleep_cycles.append(int(n * SLEEP_MS / max(e0.elapsed_time(e1), 1e-3)))
    return _sleep_cycles[0]


def _busy(s, pinned, d_in, sleep=True):
    """On stream s: SLEEP_MS of sleep, then the copy that fills the input buffer (from pinned host memory, so it really waits)."""
    import torch
    cycles = sleep_cycles()
    with torch.cuda.stream(s):
        if sleep:
            torch.cuda._sleep(cycles)
        d_in.copy_(pinned, non_blocking=True)


def _pinned(data):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(data), dtype=np.uint8).copy()).pin_memory()


def _zeros(n, dtype=None):
    import torch
    return torch.zeros(n, dtype=dtype or torch.uint8, device="cuda")


def _stage2_bufs(ctx, b):
    """Zeroed device buffers for b on slot 0 (input, out, LUT, result) and b's bytes in pinned host memory."""
    import torch
    cap = ctx.out_capacity(b.n_rec) + 64
    return (b, _zeros(b.size + 64), _zeros(cap), cap, _zeros(ctx.lut_entries, torch.int64), _zeros(8, torch.int64),
            _pinned(np.concatenate([b.data, np.zeros(64, np.uint8)])))


def _stage2_dev(ctx, bufs, s, sleep=True):
    """dev_process_bin behind a sleep and its input's copy on s."""
    b, d_bin, d_out, cap, d_lut, d_res, pinned = bufs
    _busy(s, pinned, d_bin, sleep)
    ctx.dev_process_bin(0, d_bin.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_out.data_ptr(), cap, d_lut.data_ptr(), d_res.data_ptr(), s.cuda_stream)
    return d_out, d_lut, d_res


def _dev_result(ctx, d_out, d_lut, d_res):
    r = d_res.cpu().numpy().view(np.uint64)
    assert int(r[5]) == 0 and int(r[6]) == 0, r
    return d_out[:int(r[4]) * ctx.out_rec_bytes].cpu().numpy().tobytes(), d_lut.cpu().numpy().view(np.uint64), tuple(int(x) for x in r[:4])


def test_stage2_device_forms_on_a_busy_stream(oracle):
    """dev_process_bin, and dev_expand -> dev_sort(hist_ready) -> dev_count, each queued behind a sleep and the copy of its input on the
    caller's stream, their outputs copied by torch on that stream, one synchronisation at the end: the oracle's bytes."""
    import torch
    p = _params(31, True)
    b = _bins_for(31, False)[2]
    want = _expected(oracle, 31, True, False)[2]
    ctx = Stage2Context(s2params(p))
    try:
        bufs = _stage2_bufs(ctx, b)
        _, d_bin2, d_out2, cap, d_lut2, d_res2, pinned2 = _stage2_bufs(ctx, b)
        d_recs, d_tmp = _zeros((b.n_rec + 8) * p.words, torch.int64), _zeros((b.n_rec + 8) * p.words, torch.int64)
        d_res_e = _zeros(8, torch.int64)
        torch.cuda.synchronize()
        s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        d_out, d_lut, d_res = _stage2_dev(ctx, bufs, s)
        with torch.cuda.stream(s):
            outs = [d_out.clone(), d_lut.clone(), d_res.clone()]
        # the three stages, on another busy stream (and after the call above: the same slot)
        _busy(s2, pinned2, d_bin2)
        ctx.dev_expand(0, d_bin2.data_ptr(), b.size, b.n_rec, b.pack_bytes, d_recs.data_ptr(), d_res_e.data_ptr(), s2.cuda_stream)
        where = ctx.dev_sort(0, d_recs.data_ptr(), d_tmp.data_ptr(), b.n_rec, hist_ready=True, stream=s2.cuda_stream)
        ctx.dev_count(0, (d_tmp if where else d_recs).data_ptr(), b.n_rec, d_out2.data_ptr(), cap, d_lut2.data_ptr(), d_res2.data_ptr(), s2.cuda_stream)
        with torch.cuda.stream(s2):
            outs2 = [d_out2.clone(), d_lut2.clone(), d_res2.clone()]
        torch.cuda.synchronize()
        same(_dev_result(ctx, *outs), want, "dev_process_bin")
        assert int(d_res_e.cpu()[6]) == 0
        same(_dev_result(ctx, *outs2), want, "dev_expand -> dev_sort -> dev_count")
        same(host_result(ctx.process_bin(to_skb(b))), want, "process_bin")
    finally:
        ctx.close()


def test_stage2_slot_orders_device_and_host_forms(oracle):
    """On slot 0: dev_process_bin on a sleeping stream, then dev_process_bin on an idle stream: the second ends after the first.  Again
    dev_process_bin on the sleeping stream, then process_bin: it returns after the device form has run.  All four give the oracle's bytes."""
    import torch
    b, b2 = _bins_for(31, False)[2], _bins_for(31, False)[3]
    want, want2 = _expected(oracle, 31, True, False)[2], _expected(oracle, 31, True, False)[3]
    ctx = Stage2Context(s2params(_params(31, True)))
    try:
        bufs, bufs2, bufs3 = _stage2_bufs(ctx, b), _stage2_bufs(ctx, b2), _stage2_bufs(ctx, b2)
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        first = _stage2_dev(ctx, bufs, s1)
        second = _stage2_dev(ctx, bufs2, s2, sleep=False)
        ev2 = torch.cuda.Event()
        ev2.record(s2)
        ev2.synchronize()
        assert s1.query(), "the slot's second device-form call ended before its first had run"
        third = _stage2_dev(ctx, bufs3, s1)
        r = ctx.process_bin(to_skb(b))
        assert s1.query(), "process_bin returned before the slot's device-form call had run"
        torch.cuda.synchronize()
        same(host_result(r), want, "process_bin after a device form")
        same(_dev_result(ctx, *first), want, "first dev_process_bin")
        same(_dev_result(ctx, *second), want2, "second dev_process_bin")
        same(_dev_result(ctx, *third), want2, "third dev_process_bin")
    finally:
        ctx.close()


@pytest.mark.parametrize("host_form", ["split_raw", "split_fastx"])
def test_splitter_device_form_on_a_busy_stream_then_host_form(host_form):
    """dev_split behind a sleep and its input's copy; then split_raw, or split_fastx of a FASTQ chunk, on the same splitter: it returns only
    after the device form has run (they share the workspace), and both equal the stage-1 oracle."""
    import torch
    s1o = Stage1Oracle()
    K, SIG, NB = 31, 9, 64
    sig_map = random_map(6, SIG, NB)
    batch = _batches(300, 1)[0]
    raw2 = b"".join(b"@r%d\n%s\n+\n%s\n" % (i, r, b"I" * len(r)) for i, r in enumerate(make_reads(310, "short", n_reads=120, read_len=200)))
    batch2 = _batches(310, 1)[0] if host_form == "split_raw" else sequences_to_batch(raw2).tobytes()
    want, want2 = s1o.split(batch, K, SIG, sig_map, NB), s1o.split(batch2, K, SIG, sig_map, NB)
    sp = kmc_b200.Splitter(K, SIG, sig_map, n_bins=NB, max_batch_bytes=max(len(batch), len(batch2), len(raw2) + 1))
    px = kmc_b200.FastxParser("fastq", max_chunk_bytes=len(raw2))
    try:
        cap, pcap = len(batch) * 2 + 4096, len(batch) // 64 + 4 * NB
        d_seq, d_out, d_pk = _zeros(len(batch)), _zeros(cap), _zeros(pcap, torch.int64)
        d_fr, d_res = _zeros(NB * 5, torch.int64), _zeros(5, torch.int64)
        pinned = _pinned(batch)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        _busy(s, pinned, d_seq)
        sp.dev_split(d_seq.data_ptr(), len(batch), d_out.data_ptr(), cap, d_pk.data_ptr(), pcap, d_fr.data_ptr(), d_res.data_ptr(), s.cuda_stream)
        if host_form == "split_raw":
            o2, pk2, fr2 = sp.split_raw(batch2)
        else:
            o2, pk2, fr2, used, n = sp.split_fastx(px, raw2)
            assert (used, n) == (len(raw2), len(batch2))
        assert s.query(), "%s returned before the splitter's device-form call had run" % host_form
        with torch.cuda.stream(s):
            outs = [d_out.clone(), d_pk.clone(), d_fr.clone(), d_res.clone()]
        torch.cuda.synchronize()
        res = outs[3].cpu().numpy().view(np.uint64)
        assert int(res[2]) == 0 and int(res[0]) == want.out.size and int(res[1]) == want.pack_bytes.size
        assert outs[0][:int(res[0])].cpu().numpy().tobytes() == want.out.tobytes()
        assert np.array_equal(outs[1][:int(res[1])].cpu().numpy().view(np.uint64), want.pack_bytes)
        fr = outs[2].cpu().numpy().view(np.uint64).reshape(NB, 5)          # kmcb200_bin_fragment: 4 x u64, then pack0, n_packs as u32
        assert np.array_equal(fr[:, :4], want.frags[:, :4])
        assert np.array_equal(fr[:, 4:].copy().view(np.uint32).astype(np.uint64), want.frags[:, 4:6])
        assert o2.tobytes() == want2.out.tobytes() and np.array_equal(pk2, want2.pack_bytes)
        assert np.array_equal(np.array([(f.byte_off, f.bytes, f.n_rec, f.n_super_kmers, f.pack0, f.n_packs) for f in fr2], dtype=np.uint64), want2.frags)
    finally:
        sp.close()
        px.close()


def _sparse(c):
    return c.index.tobytes(), c.value.tobytes()


# kind -> (make the handle, the oracle's counters of a list of batches, the handle's counters as compared)
COUNTERS = {
    "sigstats": (lambda mx: kmc_b200.SignatureStats(31, 9, max_batch_bytes=mx),
                 lambda bs: sum(oracle_signature_stats(b, 31, 9).astype(np.uint64) for b in bs).astype(np.uint32).tobytes(), lambda c: c.tobytes()),
    "smallk": (lambda mx: kmc_b200.SmallKCounter(11, max_batch_bytes=mx), lambda bs: sum(M.counts(np.frombuffer(b, np.uint8), 11) for b in bs).tobytes(), lambda c: c.tobytes()),
    "estimator": (lambda mx: kmc_b200.HistogramEstimator(31, max_batch_bytes=mx),
                  lambda bs: _sparse(et.SparseCounters(np.concatenate([et.oracle_increments(b, 31, 7) for b in bs]))),
                  lambda c: _sparse(et.SparseCounters.from_dense(c.reshape(-1)))),
}


@pytest.mark.parametrize("kind", list(COUNTERS))
def test_counting_handle_on_a_busy_stream_and_across_streams(kind):
    """dev_add behind a sleep and its input's copy, then read(): the batch is counted.  Then dev_add on a sleeping S1 and dev_add on S2
    (not sleeping), then read(): the counters hold both batches, because the S2 call is queued after the handle's earlier work."""
    import torch
    make, model, view = COUNTERS[kind]
    a, b = _batches(400, 2)
    want_a, want_ab = model([a]), model([a, b])
    h = make(max(len(a), len(b)))
    try:
        d_a, d_b = _zeros(len(a)), _zeros(len(b))
        pa, pb = _pinned(a), _pinned(b)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        _busy(s, pa, d_a)
        h.dev_add(d_a.data_ptr(), len(a), s.cuda_stream)
        assert view(h.read()) == want_a, "device form on a busy stream"
        h.reset()
        d_a.zero_()
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        _busy(s1, pa, d_a)
        h.dev_add(d_a.data_ptr(), len(a), s1.cuda_stream)
        with torch.cuda.stream(s2):
            d_b.copy_(pb, non_blocking=True)
        h.dev_add(d_b.data_ptr(), len(b), s2.cuda_stream)
        assert view(h.read()) == want_ab, "two streams"
    finally:
        h.close()


def test_parser_device_form_on_a_busy_stream_then_host_form():
    """dev_parse behind a sleep and its input's copy, its output copied on that stream; then parse() on the same parser returns only after
    the device form has run (they share the tile summaries); both equal sequences_to_batch."""
    import torch
    raw, raw2 = fastq_text(500, 400), fastq_text(501, 300)
    px = kmc_b200.FastxParser("fastq", max_chunk_bytes=max(len(raw), len(raw2)))
    try:
        d_raw, d_seq, d_res = _zeros(len(raw)), _zeros(len(raw) + 1), _zeros(4, torch.int64)
        pinned = _pinned(raw)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        _busy(s, pinned, d_raw)
        px.dev_parse(d_raw.data_ptr(), len(raw), True, None, d_seq.data_ptr(), len(raw) + 1, d_res.data_ptr(), s.cuda_stream)
        seq2, used2 = px.parse(raw2)
        assert s.query(), "parse returned before the parser's device-form call had run"
        with torch.cuda.stream(s):
            outs = [d_seq.clone(), d_res.clone()]
        torch.cuda.synchronize()
        r = outs[1].cpu().numpy().view(np.uint64)
        assert int(r[3]) == 0 and int(r[0]) == len(raw)
        assert outs[0][:int(r[1])].cpu().numpy().tobytes() == sequences_to_batch(raw).tobytes()
        assert seq2.tobytes() == sequences_to_batch(raw2).tobytes() and used2 == len(raw2)
    finally:
        px.close()


def test_inflater_device_form_on_a_busy_stream():
    """dev_inflate behind a sleep and the copy of the compressed members, its text copied on that stream: zlib's text."""
    import torch
    text = b"".join(fastq_text(600 + i, 200) for i in range(3))
    raw = bgzf(text, seed=3)
    _, t, m = kmc_b200.bgzf_scan(raw, 1 << 40)
    gz = kmc_b200.Gunzip(0, 1 << 22, 1 << 22)
    try:
        d_raw, d_m, d_text, d_err = _zeros(len(raw)), torch.from_numpy(m.view(np.uint8).copy()).cuda(), _zeros(t), _zeros(1, torch.int64)
        pinned = _pinned(raw)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        _busy(s, pinned, d_raw)
        gz.dev_inflate(d_m.data_ptr(), len(m), d_raw.data_ptr(), len(raw), d_text.data_ptr(), t, d_err.data_ptr(), s.cuda_stream)
        with torch.cuda.stream(s):
            outs = [d_text.clone(), d_err.clone()]
        torch.cuda.synchronize()
        assert int(outs[1].item()) == -1
        assert outs[0].cpu().numpy().tobytes() == inflate_all(raw) == text
    finally:
        gz.close()
