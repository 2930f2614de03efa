"""KMC database input on the host: the header parse and its refusals, the numpy model of the reader (kmc_db_to_batch) against the batches
the reference read, the InitKMC signature map against the map the reference's output implies, and the prefix rule on synthetic LUTs."""
import hashlib
import json
import os
import struct

import numpy as np
import pytest

from kmc_input_testlib import CASES, INPUT_DBS, KMC_INPUT_GOLDEN, materialize
from kmc_b200 import KmcB200Error
from kmc_b200.reads import (KMC1_VERSION, KMC2_VERSION, _kmc_inputs, kmc_db_info, kmc_db_to_batch, kmc_input_signature_map, kmc_records_to_batch,
                            predicted_size, signature_map_from_kmc_pre)

GOLDEN = json.load(open(KMC_INPUT_GOLDEN))


@pytest.fixture(scope="module")
def dbs(tmp_path_factory):
    return materialize(tmp_path_factory.mktemp("kmc_input"))


def test_header_of_every_input_database(dbs):
    for name, (_, _, _, k, opts) in INPUT_DBS.items():
        info = kmc_db_info(dbs[name])
        assert info.kmer_len == k
        assert info.version == (KMC1_VERSION if k <= 13 else KMC2_VERSION)
        assert info.lut[0] == 0 and np.all(np.diff(info.lut.astype(np.int64)) >= 0)
        assert int(info.lut[-1]) == info.total_kmers
        assert os.path.getsize(dbs[name] + ".kmc_suf") == 8 + info.total_kmers * info.record_bytes
        if info.version == KMC2_VERSION:
            assert info.signature_len == 5 and info.n_bins == 64
            assert info.lut.size == info.n_bins * 4 ** info.lut_prefix_len + 1
        else:
            assert info.lut.size == 4 ** info.lut_prefix_len + 1
    assert kmc_db_info(dbs["k31_cs1"]).counter_size == 0
    assert kmc_db_info(dbs["k31_cs2"]).counter_size == 2
    assert kmc_db_info(dbs["k31_cs3"]).counter_size == 3 and kmc_db_info(dbs["k31_cs3"]).max_count == 100000
    assert kmc_db_info(dbs["k31_cs4"]).counter_size == 4
    assert kmc_db_info(dbs["k31_ci5_cs3"]).min_count == 5


@pytest.mark.parametrize("name", sorted(CASES))
def test_model_batch_is_what_the_reference_read(dbs, name):
    inputs = CASES[name][0]
    batch = np.concatenate([kmc_db_to_batch(dbs[i]) for i in inputs])
    assert hashlib.md5(batch.tobytes()).hexdigest() == GOLDEN["cases"][name]["batch_md5"]
    if "n_reads" in GOLDEN["cases"][name]:
        assert int(np.count_nonzero(batch == 10)) == GOLDEN["cases"][name]["n_reads"]


def test_filtered_database_reads_nothing(dbs):
    assert kmc_db_info(dbs["k31_ci5_cs3"]).total_kmers > 0 and kmc_db_to_batch(dbs["k31_ci5_cs3"]).size == 0
    info = kmc_db_info(dbs["k31_cs1"])
    assert kmc_db_to_batch(dbs["k31_cs1"]).size == info.total_kmers * 32


def _patched(dbs, tmp_path, name, patch):
    src = dbs[name]
    pre = bytearray(open(src + ".kmc_pre", "rb").read())
    for at, b in patch.items():
        pre[len(pre) + at:len(pre) + at + len(b)] = b
    out = str(tmp_path / ("patched_" + name))
    open(out + ".kmc_pre", "wb").write(pre)
    open(out + ".kmc_suf", "wb").write(open(src + ".kmc_suf", "rb").read())
    return out


def test_header_refusals(dbs, tmp_path):
    with pytest.raises(KmcB200Error, match="neither KMC1"):
        kmc_db_info(_patched(dbs, tmp_path, "k31", {-12: struct.pack("<I", 0x100)}))
    pre = open(dbs["k31"] + ".kmc_pre", "rb").read()
    h = len(pre) - 8 - struct.unpack_from("<I", pre, len(pre) - 8)[0]
    with pytest.raises(KmcB200Error, match="Quake"):
        kmc_db_info(_patched(dbs, tmp_path, "k31", {h + 4 - len(pre): struct.pack("<I", 1)}))
    with pytest.raises(KmcB200Error, match="counters of 5 bytes"):
        kmc_db_info(_patched(dbs, tmp_path, "k31", {h + 8 - len(pre): struct.pack("<I", 5)}))
    with pytest.raises(KmcB200Error, match="KMCP"):
        kmc_db_info(_patched(dbs, tmp_path, "k31", {-4: b"XXXX"}))


def test_refusals_carry_the_reference_messages(dbs):
    msgs = GOLDEN["refusals"]
    with pytest.raises(KmcB200Error, match=msgs["kmc1_on_bin_path"].split(".")[0]):
        kmc_input_signature_map(dbs["k10_kmc1"], 9)
    with pytest.raises(KmcB200Error, match=msgs["signature_len"]):
        kmc_input_signature_map(dbs["k31"], 7, 64)
    with pytest.raises(KmcB200Error, match=msgs["n_bins"]):
        kmc_input_signature_map(dbs["k31"], 5, 256)
    with pytest.raises(KmcB200Error) as e:
        kmc_input_signature_map(dbs["k10_kmc1"], 9)
    assert str(e.value).endswith(msgs["kmc1_on_bin_path"])


def test_input_kinds_are_not_mixed(dbs, tmp_path):
    fq = tmp_path / "r.fq"
    fq.write_bytes(b"@r\nACGT\n+\nIIII\n")
    assert _kmc_inputs([dbs["k31"], dbs["k25"]]) and not _kmc_inputs([str(fq)])
    with pytest.raises(KmcB200Error, match="every input"):
        _kmc_inputs([dbs["k31"], str(fq)])


def test_predicted_size_is_the_last_databases_total(dbs):
    a, b = kmc_db_info(dbs["k31"]).total_kmers, kmc_db_info(dbs["k25"]).total_kmers
    assert predicted_size([dbs["k31"], dbs["k25"]]) == b and predicted_size([dbs["k25"], dbs["k31"]]) == a


def _init_kmc(stored, n_bins):
    """CSignatureMapper::InitKMC's loop, literally."""
    groups = {}
    for sig, v in enumerate(stored):
        groups.setdefault(int(v), []).append(sig)
    out, bin_no, special = [0] * len(stored), 0, len(stored) - 1
    for v in sorted(groups):
        was_special = False
        for sig in groups[v]:
            if sig == special:
                was_special = True
                out[sig] = n_bins - 1
            else:
                out[sig] = bin_no
        if not was_special:
            bin_no += 1
    return np.array(out)


@pytest.mark.parametrize("name", ["k31", "k25", "k55", "k128"])
def test_signature_map_is_init_kmc(dbs, name):
    info = kmc_db_info(dbs[name])
    bins, n_bins = kmc_input_signature_map(dbs[name], 5)
    assert n_bins == 64 and np.array_equal(bins, _init_kmc(info.signature_map, n_bins))
    rng = np.random.default_rng(5)                                      # a special signature inside a group, and shared values
    stored = rng.integers(0, 40, info.signature_map.size).astype(np.uint32)
    info.signature_map = stored
    from kmc_b200 import reads
    orig = reads.kmc_db_info
    try:
        reads.kmc_db_info = lambda p: info
        bins, _ = kmc_input_signature_map(dbs[name], 5)
    finally:
        reads.kmc_db_info = orig
    assert np.array_equal(bins, _init_kmc(stored, 64))


def test_signature_map_matches_the_reference_output(dbs, tmp_path):
    """The database stores every signature's bin file position: the signatures of one InitKMC bin share one position."""
    bins, _ = kmc_input_signature_map(dbs["k31"], 5)
    _, stored = signature_map_from_kmc_pre(dbs["k31"] + ".kmc_pre")
    for b in np.unique(bins):
        assert np.unique(stored[bins == b]).size == 1 or b == 63


class _Info:
    def __init__(self, k, lp, cs, lut, total, min_count=0, max_count=(1 << 32) - 1):
        self.kmer_len, self.lut_prefix_len, self.counter_size = k, lp, cs
        self.suffix_bytes = (k - lp) // 4
        self.record_bytes = self.suffix_bytes + cs
        self.lut = np.asarray(lut, dtype=np.uint64)
        self.total_kmers, self.min_count, self.max_count = total, min_count, max_count


def _brute_prefix(lut, g, lp):
    return sum(1 for j in range(1, len(lut)) if int(lut[j]) <= g) & ((1 << (2 * lp)) - 1)


def _prefixes(info, first, n):
    batch = kmc_records_to_batch(info, np.zeros((n, info.record_bytes), dtype=np.uint8), first).reshape(n, info.kmer_len + 1)
    code = {65: 0, 67: 1, 71: 2, 84: 3}
    return [sum(code[int(c)] << (2 * (info.lut_prefix_len - 1 - i)) for i, c in enumerate(row[:info.lut_prefix_len])) for row in batch]


def test_prefix_rule_on_synthetic_luts():
    # empty prefixes everywhere but a few, two bins (the prefix wraps), and a KMC1 guard
    lut = [0, 0, 0, 5, 5, 5, 5, 9, 9, 9, 9, 9, 9, 9, 12, 12, 12, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20, 20]
    info = _Info(6, 2, 0, lut[:33], 20)
    assert _prefixes(info, 0, 20) == [_brute_prefix(info.lut, g, 2) for g in range(20)]
    kmc1 = _Info(6, 2, 0, [0, 3, 3, 7] + [0] * 12 + [10], 10)          # the stored words, then total_kmers
    kmc1.lut = np.array([0, 3, 3, 7, 8, 8, 8, 8, 8, 8, 9, 9, 9, 9, 9, 9, 10], dtype=np.uint64)
    assert _prefixes(kmc1, 0, 10) == [_brute_prefix(kmc1.lut, g, 2) for g in range(10)]


def test_prefix_rule_past_two_to_the_32():
    base = (1 << 32) + 7
    lut = np.array([0] + [base - 3, base + 1, base + 1, base + 2] + [base + 100] * 12, dtype=np.uint64)
    info = _Info(6, 2, 0, lut, base + 100)
    assert _prefixes(info, base - 5, 10) == [_brute_prefix(lut, g, 2) for g in range(base - 5, base + 5)]


def test_counter_filter_is_uint32():
    info = _Info(8, 4, 4, [0] * 256 + [4], 4, min_count=2, max_count=0xFFFFFFFF)
    recs = np.array([[0x1B, 1, 0, 0, 0], [0x1B, 2, 0, 0, 0], [0xE4, 0xFF, 0xFF, 0xFF, 0xFF], [0x00, 0, 0, 0, 1]], dtype=np.uint8)
    batch = kmc_records_to_batch(info, recs, 0)
    assert batch.tobytes() == b"TTTTACGT\nTTTTTGCA\nTTTTAAAA\n"
