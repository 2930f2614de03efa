"""The database writer of SURVEY 8f N3 (kmcb200_db_*: pinned staging ring, writer thread, footer) against files written by the REFERENCE:
a database made by the unmodified reference CLI (one stage-2 sorter so that the bin order is deterministic; stored in
tests/golden/refdb_k*.npz by tests/golden/make_reference_digests.py) is taken apart into its bins (payload and LUT of every bin, signature
map, header fields) and replayed through the writer; .kmc_pre and .kmc_suf must come out byte for byte.  Host-only: runs without a GPU
(the staging ring is then plain memory)."""
import os
import struct

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
# the reference CLI's runs behind tests/golden/refdb_k<k>.npz: 200 reads of tests/test_gpu_kmc_files.write_fastq(seed 500 + k,
# genome_len=2000, err=0.002), `kmc -k<k> -fq -m2 -t4 -sr1 -n64 <extra>`
REFDB_CASES = {31: ("-ci2",), 28: ("-ci1", "-cs65535"), 55: ("-ci1", "-b")}
REFDB_STATS = ("#Unique_k-mers", "#k-mers_below_min_threshold", "#k-mers_above_max_threshold", "#Total no. of k-mers")


def load_reference_db(k, tmp):
    """The stored reference database of REFDB_CASES[k] as <tmp>/ref.kmc_pre / .kmc_suf, and its statistics."""
    z = np.load(os.path.join(GOLD, "refdb_k%d.npz" % k))
    db = os.path.join(tmp, "ref")
    for ext in ("kmc_pre", "kmc_suf"):
        with open(db + "." + ext, "wb") as f:
            f.write(z[ext].tobytes())
    return db, dict(zip(REFDB_STATS, (int(x) for x in z["stats"])))


def parse_db(prefix):
    pre = open(prefix + ".kmc_pre", "rb").read()
    suf = open(prefix + ".kmc_suf", "rb").read()
    assert pre[:4] == b"KMCP" and pre[-4:] == b"KMCP" and suf[:4] == b"KMCS" and suf[-4:] == b"KMCS"
    header_offset = struct.unpack("<I", pre[-8:-4])[0]
    h = len(pre) - 8 - header_offset
    k, mode, counter_size, p, sig_len, cmin, cmax = struct.unpack("<7I", pre[h:h + 28])
    n_counted, = struct.unpack("<Q", pre[h + 28:h + 36])
    both = pre[h + 36] == 0
    map_entries = (1 << (2 * sig_len)) + 1
    m0 = h - 4 * map_entries
    sig_map = np.frombuffer(pre[m0:h], dtype=np.uint32)
    n_recs, = struct.unpack("<Q", pre[m0 - 8:m0])
    lut_all = np.frombuffer(pre[4:m0 - 8], dtype=np.uint64)
    n_lut = 1 << (2 * p)
    assert lut_all.size % n_lut == 0
    luts = lut_all.reshape(-1, n_lut)
    rec = (k - p) // 4 + counter_size
    starts = np.append(luts[:, 0], np.uint64(n_recs)).astype(np.int64)
    payloads = [suf[4 + int(starts[b]) * rec:4 + int(starts[b + 1]) * rec] for b in range(luts.shape[0])]
    assert 4 + n_recs * rec + 4 == len(suf)
    return dict(k=k, counter_size=counter_size, p=p, sig_len=sig_len, cmin=cmin, cmax=cmax, both=both, n_counted=n_counted,
                sig_map=sig_map, luts=luts, payloads=payloads, n_recs=n_recs)


@pytest.mark.parametrize("k,extra", list(REFDB_CASES.items()))
@pytest.mark.parametrize("raw_lut", [False, True])
def test_writer_reproduces_reference_files(tmp_path, k, extra, raw_lut):
    import ctypes as C
    import kmc_b200
    tmp = str(tmp_path)
    db, st = load_reference_db(k, tmp)
    d = parse_db(db)
    out = os.path.join(tmp, "replay")
    w = kmc_b200.DbWriter(out, d["k"], d["counter_size"], d["p"], d["sig_len"], d["cmin"], d["cmax"], d["both"], staging_bytes=1 << 20)   # the smallest ring (1 MB); the standalone tests below make it wrap
    n_bins = d["luts"].shape[0]
    for b in range(n_bins):
        pay = d["payloads"][b]
        ptr = w.reserve(len(pay))
        C.memmove(ptr, pay, len(pay))
        lut = d["luts"][b]
        if raw_lut:
            nxt = np.append(lut[1:], np.uint64(w.records + len(pay) // max((d["k"] - d["p"]) // 4 + d["counter_size"], 1)))
            lut = nxt - lut
        # the statistics only enter the file as n_unique - n_cutoff_min - n_cutoff_max: give them all to the first bin
        bin_stats = (int(st["#Unique_k-mers"]), int(st["#k-mers_below_min_threshold"]), int(st["#k-mers_above_max_threshold"]), int(st["#Total no. of k-mers"])) if b == 0 else (0, 0, 0, 0)
        sigs = np.nonzero(d["sig_map"] == b)[0]
        w.commit_bin(len(pay), lut, bin_stats, sigs, raw_lut=raw_lut)
    tot = w.close()
    assert tot[0] - tot[1] - tot[2] == d["n_counted"]
    assert open(out + ".kmc_suf", "rb").read() == open(db + ".kmc_suf", "rb").read()
    assert open(out + ".kmc_pre", "rb").read() == open(db + ".kmc_pre", "rb").read()


def _standalone_bins():
    from kmc_testlib import synth_bin
    sizes = [4000, 0, 900, 15000, 1, 7000, 200000]          # the last bin alone emits > 1 MB of records: the 1 MB staging ring wraps and blocks
    return [synth_bin(40 + i, 31, n, genome_len=max(n, 500)) for i, n in enumerate(sizes)]


RING_BYTES = 1 << 20                # kmcb200_db_open's smallest staging ring (db_writer.inl), what the tests below ask for


def write_standalone(out, results, p):
    """Oracle results -> the writer (raw LUTs, bin i holds signature i) -> out.kmc_pre / out.kmc_suf; returns the totals."""
    import ctypes as C
    import kmc_b200
    w = kmc_b200.DbWriter(out, p.k, p.counter_bytes, p.lut_prefix_len, 9, p.cutoff_min, p.cutoff_max, True, staging_bytes=RING_BYTES)
    for i, r in enumerate(results):
        ptr = w.reserve(len(r.payload))
        C.memmove(ptr, r.payload, len(r.payload))
        w.commit_bin(len(r.payload), r.lut, r.stats, [i], raw_lut=True)
    return w.close()


def db_digest(prefix):
    from kmc_testlib import digest
    return {ext: digest(open(prefix + ext, "rb").read()) for ext in (".kmc_pre", ".kmc_suf")}


def _assert_reference_readable(out, case, results, p):
    """The files are byte for byte the ones the reference's kmc_tools read back to the expected dump when the digests were stored
    (tests/golden/make_reference_digests.py), and this file's reader decodes them to the same dump."""
    from kmc_testlib import reference_digest, decode_payload
    assert db_digest(out) == reference_digest(case)["results"]["kmc_tools_read_back"]
    d = parse_db(out)
    ends = np.append(d["luts"][1:, 0], np.uint64(d["n_recs"]))
    decoded = []
    for b, pay in enumerate(d["payloads"]):
        counts = np.diff(np.append(d["luts"][b], ends[b]).astype(np.int64))
        decoded += ["%s\t%d" % (s, c) for s, c in decode_payload(pay, counts, p)]
    assert decoded == _expected_dump(results, p)


def _expected_dump(results, p):
    from kmc_testlib import decode_payload
    lines = []
    for r in results:
        lines += ["%s\t%d" % (s, c) for s, c in decode_payload(r.payload if isinstance(r.payload, bytes) else r.payload.tobytes(), r.lut, p)]
    return lines


def test_standalone_database_is_readable_by_the_reference_tools(tmp_path, oracle):
    """Bins -> (oracle results) -> writer -> files that the reference's kmc_tools reads back bin after bin."""
    from kmc_testlib import Params
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    res = [oracle.process_bin(b, p) for b in _standalone_bins()]
    out = os.path.join(str(tmp_path), "standalone")
    assert sum(len(r.payload) for r in res) > RING_BYTES
    tot = write_standalone(out, res, p)
    assert tot == tuple(sum(r.stats[j] for r in res) for j in range(4))
    _assert_reference_readable(out, "standalone_db", res, p)


@pytest.mark.gpu
def test_gpu_bins_straight_into_the_database(tmp_path, oracle):
    """The standalone stage 2: bins -> kmcb200_submit_bin with the writer's pinned ring as D2H target -> kmcb200_wait_bin_scanned (LUT prefix
    sum on the GPU, base = records so far) -> commit; two bins in flight while the writer thread appends the earlier ones."""
    import kmc_b200
    from kmc_testlib import Params
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    bins = _standalone_bins() * 3
    res = [oracle.process_bin(b, p) for b in bins]
    out = os.path.join(str(tmp_path), "gpu_db")
    ctx = kmc_b200.Stage2Context(kmc_b200.Stage2Params(31, True, 2, 10 ** 9, 255, 7), device=0, n_slots=2)
    w = kmc_b200.DbWriter(out, 31, p.counter_bytes, 7, 9, p.cutoff_min, p.cutoff_max, True, staging_bytes=RING_BYTES)
    luts = [np.zeros(ctx.lut_entries, dtype=np.uint64) for _ in range(2)]
    datas = [np.ascontiguousarray(b.data) for b in bins]

    def finish(i):
        nbytes, stats = ctx.wait_bin_scanned(i % 2, w.records)
        assert stats == res[i].stats and nbytes == len(res[i].payload)
        w.commit_bin(nbytes, luts[i % 2], stats, [i])

    # one region is open at a time (commit order = file order), so the pipeline is: reserve i, submit i, (GPU works), wait i, commit i -
    # the overlap is between the GPU / the copies of bin i and the writer thread's fwrite of bins < i
    for i, b in enumerate(bins):
        cap = ctx.out_capacity(b.n_rec) + 64
        ptr = w.reserve(cap)
        ctx.submit_bin(i % 2, datas[i].ctypes.data, datas[i].size, b.n_rec, np.ascontiguousarray(b.pack_bytes), ptr, cap, luts[i % 2].ctypes.data)
        finish(i)
    tot = w.close()
    ctx.close()
    assert tot == tuple(sum(r.stats[j] for r in res) for j in range(4))
    _assert_reference_readable(out, "standalone_db_x3", res, p)
