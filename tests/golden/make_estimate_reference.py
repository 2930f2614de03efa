"""Writes tests/golden/estimate_reference.json: what the reference's histogram estimator gives on seeded inputs, as MD5s of the `kmc -e`
text file (kmc_CLI/kmc.cpp:308-321), plus the generator parameters of every input (tests/estimate_testlib.py rebuilds them).

    python tests/golden/make_estimate_reference.py        # needs oracle/_ref/kmc_ref and oracle/_ref/libkmc_nthash_ref.so (build())

  cli      `kmc_ref -e` on FASTQ and on multi-line FASTA (-fm) of the same reads, k from 1 to 256, and on the corner inputs
  harness  the reference's CntHashEstimator itself (oracle/ref/nthash_harness.cpp) at every k = 1..256 with s = 7, and with s = 11, which
           the CLI takes only for inputs of at least 5 * 10^10 bytes
  db       MD5s of the `kmc_ref -sr1` database files with and without --opt-out-size (the LUT prefix length chosen from the estimate)
"""
import json
import os
import subprocess
from concurrent.futures import ProcessPoolExecutor
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import estimate_testlib as et  # noqa: E402

KMC_REF = os.path.join(et.ROOT, "oracle", "_ref", "kmc_ref")
CLI_KS = [1, 5, 13, 21, 25, 31, 32, 33, 55, 63, 64, 65, 127, 128, 129, 200, 256]
LONG = {"kind": "reads", "seed": 4401, "n_reads": 3000, "read_len": [260, 700]}
HARNESS_INPUT = {"kind": "reads", "seed": 4402, "n_reads": 400, "read_len": [260, 600], "lower_frac": 0.05}


def run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        raise RuntimeError("%s failed:\n%s" % (" ".join(cmd), r.stdout[-2000:]))


def kmc_e(tmp, case):
    path = os.path.join(tmp, "in." + case["format"])
    with open(path, "wb") as f:
        f.write(et.case_text(case))
    out = os.path.join(tmp, "hist.txt")
    run([KMC_REF, "-k%d" % case["k"], "-fm" if case["format"] == "fasta" else "-fq", "-t4", "-m2", "-e", path, out, tmp])
    return et.md5(open(out, "rb").read())


def sampled_kmer(k, s, seed):
    """A k-mer the estimator samples (by the oracle's hash), so that its copies land in one counter."""
    import numpy as np
    rng = np.random.default_rng(seed)
    while True:
        kmer = bytes(np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, k)])
        if et.oracle_increments(kmer + b"\n", k, s).size:
            return kmer.decode()


def harness_md5(case):
    return et.md5(et.hist_text(et.harness_histogram(et.case_batch(case), case["k"], case["s"])))


def main():
    cli, db = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for k in CLI_KS:
            for fmt in ("fastq", "fasta"):
                c = {"name": "long_k%d_%s" % (k, fmt), "k": k, "s": 7, "format": fmt, "gen": LONG}
                c["md5"] = kmc_e(tmp, c)
                cli.append(c)
        corners = [
            {"name": "n_dense_k25", "k": 25, "gen": {"kind": "reads", "seed": 4403, "n_reads": 2000, "read_len": 300, "n_frac": 0.05}},
            {"name": "shorter_than_k_k31", "k": 31, "gen": {"kind": "reads", "seed": 4404, "n_reads": 3000, "read_len": [10, 30]}},
            {"name": "empty_k21", "k": 21, "gen": {"kind": "empty"}},
            {"name": "max_occ_k21", "k": 21, "gen": {"kind": "repeat", "kmer": sampled_kmer(21, 7, 4405), "copies": 70000, "seed": 4406,
                                                     "n_reads": 200, "read_len": 300}},
        ]
        for c in corners:
            c.update(s=7, format="fastq")
            try:
                c["md5"] = kmc_e(tmp, c)
            except RuntimeError:
                if c["gen"]["kind"] != "empty":
                    raise
                c["md5"] = None                                       # the CLI refuses an empty input: the harness case below pins it
            cli.append(c)
        harness = [{"name": "harness_k%d_s%d" % (k, s), "k": k, "s": s, "format": "fastq", "gen": HARNESS_INPUT}
                   for s, ks in ((7, range(1, 257)), (11, (21, 31, 55, 128))) for k in ks]
        with ProcessPoolExecutor(8) as pool:                           # each call holds the reference's 1 GiB of counters
            for c, m in zip(harness, pool.map(harness_md5, harness)):
                c["md5"] = m
        harness.append({"name": "harness_empty_k21", "k": 21, "s": 7, "format": "fastq", "gen": {"kind": "empty"},
                        "md5": et.md5(et.hist_text(et.harness_histogram(b"", 21, 7)))})
        for name, k, fmt, gen, extra in (
                ("lp_changes_k30", 30, "fastq", {"kind": "reads", "seed": 4410, "n_reads": 100_000, "read_len": 150, "genome_len": 200_000},
                 ["-n64", "-ci1"]),
                ("lp_same_k25", 25, "fastq", {"kind": "reads", "seed": 4411, "n_reads": 20_000, "read_len": 150, "genome_len": 2_000_000},
                 ["-n64", "-ci2"]),
                ("fasta_k31", 31, "fasta", {"kind": "reads", "seed": 4412, "n_reads": 4000, "read_len": [200, 500]}, ["-n64", "-ci1"])):
            c = {"name": name, "k": k, "format": fmt, "gen": gen, "args": extra}
            path = os.path.join(tmp, "in." + fmt)
            with open(path, "wb") as f:
                f.write(et.case_text(c))
            for opt in (False, True):
                out = os.path.join(tmp, "db")
                run([KMC_REF, "-k%d" % k, "-fm" if fmt == "fasta" else "-fq", "-t4", "-m2", "-sr1"] + extra +
                    (["--opt-out-size"] if opt else []) + [path, out, tmp])
                c["opt" if opt else "default"] = {ext: et.md5(open(out + "." + ext, "rb").read()) for ext in ("kmc_pre", "kmc_suf")}
            db.append(c)
    with open(et.GOLDEN, "w") as f:
        json.dump({"cli": cli, "harness": harness, "db": db}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
