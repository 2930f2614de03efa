"""Whole-file parity through KMC::Runner (SURVEY 8a row 9, 8c levels L1 / L2): the reference's own CLI, compiled with the
INTEGRATION.md patch (oracle/_ref/kmc_b200cli: CKmerBinSorterB200 in place of CKmerBinSorter, everything else - stage 1, bin reader,
completer, file format - the reference's unchanged code), against the unmodified reference CLI (oracle/_ref/kmc_ref) on the same FASTQ.

  L1  .kmc_pre / .kmc_suf byte-identical (md5) to the CPU build run with ONE stage-2 sorter (-sr1): with a single sorter object bins
      reach the completer in get_sorted_req_sizes order in both builds (SURVEY section 0.3: with >1 sorters the reference's own files
      differ from run to run)
  L2  `kmc_tools transform db dump -s` text identical, also with several GPU sorter objects (any completion order)
  +   the reference's CLI known-answers (.github/workflows/main.yml:35-52; the reads live in tests/golden/kats.json)

The binaries are built from a KMC source tree by `make -C oracle cli REF=<tree>` (or build() with KMC_REFERENCE_DIR=<tree>); without
them these tests skip.  Nothing here reads the KMC sources at run time.
"""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
KMC_REF, KMC_B200, KMC_TOOLS = (os.path.join(REF, n) for n in ("kmc_ref", "kmc_b200cli", "kmc_tools"))


def _need_binaries():
    for b in (KMC_REF, KMC_B200, KMC_TOOLS):
        if not os.path.exists(b):
            pytest.skip("%s not built (make -C oracle cli REF=<KMC source tree>)" % os.path.basename(b))


def write_fastq(path, seed, n_reads, read_len=150, genome_len=200_000, err=0.01, n_frac=0.002):
    """Seeded synthetic reads: random genome, both strands, substitutions, a few N (which cut super-k-mers, splitter.cpp:557-677)."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, genome_len, dtype=np.uint8)
    comp = np.array([3, 2, 1, 0], dtype=np.uint8)
    letters = np.frombuffer(b"ACGT", dtype=np.uint8)
    pos = rng.integers(0, genome_len - read_len, n_reads)
    with open(path, "wb") as f:
        for i in range(n_reads):
            r = genome[pos[i]:pos[i] + read_len].copy()
            if rng.integers(0, 2):
                r = comp[r[::-1]]
            m = rng.random(read_len) < err
            r = np.where(m, (r + rng.integers(1, 4, read_len)) % 4, r).astype(np.uint8)
            s = letters[r].copy()
            s[rng.random(read_len) < n_frac] = ord("N")
            f.write(b"@r%d\n" % i + s.tobytes() + b"\n+\n" + b"I" * read_len + b"\n")


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def run(cmd, env=None, cwd=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run(cmd, env=e, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, "%s failed:\n%s" % (" ".join(cmd), r.stdout[-3000:])
    return r.stdout


def count(binary, tmp, tag, fastq, k, extra=(), env=None, fmt="-fq"):
    out = os.path.join(tmp, "db_%s" % tag)
    wd = os.path.join(tmp, "wd_%s" % tag)
    os.makedirs(wd, exist_ok=True)
    js = os.path.join(tmp, "stats_%s.json" % tag)
    run([binary, "-k%d" % k, fmt, "-m2", "-t4", "-j" + js] + list(extra) + [fastq, out, wd], env=env)
    return out, json.load(open(js))


def dump_sorted(tmp, db, tag):
    txt = os.path.join(tmp, "dump_%s.txt" % tag)
    run([KMC_TOOLS, "transform", db, "dump", "-s", txt])
    return open(txt).read()


@pytest.mark.parametrize("k,extra", [(28, ("-ci1",)), (31, ("-ci2",)), (55, ("-ci2",)), (31, ("-ci1", "-b")), (17, ("-ci3", "-cs7"))])
def test_kmc_database_files_identical(tmp_path, k, extra):
    _need_binaries()
    tmp = str(tmp_path)
    fq = os.path.join(tmp, "reads.fq")
    write_fastq(fq, 1000 + k, 30000)
    ref_db, ref_stats = count(KMC_REF, tmp, "ref", fq, k, extra + ("-sr1",))
    gpu_db, gpu_stats = count(KMC_B200, tmp, "gpu", fq, k, extra, env={"KMC_B200_DEVICES": "0", "KMC_B200_SORTERS_PER_GPU": "1"})
    # L1: byte-identical database files
    assert md5(gpu_db + ".kmc_suf") == md5(ref_db + ".kmc_suf"), "k=%d: .kmc_suf differs" % k
    assert md5(gpu_db + ".kmc_pre") == md5(ref_db + ".kmc_pre"), "k=%d: .kmc_pre differs" % k
    for key in ("#Unique_k-mers", "#k-mers_below_min_threshold", "#k-mers_above_max_threshold", "#Unique_counted_k-mers", "#Total no. of k-mers"):
        if key in ref_stats.get("Stats", ref_stats):
            assert gpu_stats.get("Stats", gpu_stats)[key] == ref_stats.get("Stats", ref_stats)[key], key
    # L2: several sorter objects on the GPU (bins complete in any order): the sorted dump must not change
    multi_db, _ = count(KMC_B200, tmp, "gpu3", fq, k, extra, env={"KMC_B200_DEVICES": "0", "KMC_B200_SORTERS_PER_GPU": "3"})
    ref_dump = dump_sorted(tmp, ref_db, "ref")
    assert len(ref_dump) > 1000
    assert dump_sorted(tmp, gpu_db, "gpu") == ref_dump
    assert dump_sorted(tmp, multi_db, "gpu3") == ref_dump


def test_reference_cli_known_answers_through_the_patched_binary(tmp_path):
    """single_read.fq k=28 -ci1 -> 70 k-mers in total (main.yml:35-38); issue-180 palindromes k=5 -> exact dump (:48-52; small-k path)."""
    _need_binaries()
    tmp = str(tmp_path)
    kats = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "kats.json")))
    for i, kat in enumerate(kats):
        fa = os.path.join(tmp, "kat%d.fa" % i)
        with open(fa, "w") as f:
            for j, r in enumerate(kat["reads"]):
                f.write(">r%d\n%s\n" % (j, r))
        db, stats = count(KMC_B200, tmp, "kat%d" % i, fa, kat["k"], ("-ci%d" % kat["cutoff_min"],), env={"KMC_B200_DEVICES": "0"}, fmt="-fm")
        st = stats.get("Stats", stats)
        assert int(st["#Total no. of k-mers"]) == kat["n_total"]
        if "dump" in kat:
            got = [tuple(l.split()) for l in dump_sorted(tmp, db, "kat%d" % i).splitlines()]
            assert got == [(s, str(c)) for s, c in kat["dump"]]


def test_kmc_runner_on_several_gpus(tmp_path):
    """KMC_B200_DEVICES lists one sorter object per GPU, all pulling from the reference's CBinQueue (kmc.h:1564-1600): needs >= 2 GPUs."""
    import torch
    _need_binaries()
    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("one GPU visible")
    tmp = str(tmp_path)
    fq = os.path.join(tmp, "reads.fq")
    write_fastq(fq, 77, 60000)
    ref_db, _ = count(KMC_REF, tmp, "ref", fq, 31, ("-ci2", "-sr1"))
    devs = ",".join(str(i) for i in range(min(n_dev, 8)))
    gpu_db, _ = count(KMC_B200, tmp, "gpus", fq, 31, ("-ci2",), env={"KMC_B200_DEVICES": devs, "KMC_B200_SORTERS_PER_GPU": "2"})
    assert dump_sorted(tmp, gpu_db, "gpus") == dump_sorted(tmp, ref_db, "ref")
