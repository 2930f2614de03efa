"""Stores what the unmodified reference computed for the inputs of the tests that compare against it, so that those tests run
without a reference build: tests/golden/reference_digests.json, one entry per case = SHA-256 of the generated input and, per way
the reference was run, SHA-256 of the payload / LUT plus the four counters (kmc_testlib.result_digest).

Also the database files that kmcb200_db_* writes for tests/test_db_writer.py's bins, once the reference's kmc_tools has read them back
to the expected dump, (tests/golden/refdb_k*.npz) the databases the reference CLI makes from test_db_writer.REFDB_CASES, and the sorted
dump of what the reference CLI counts in test_reference_cli's FASTQ.

Needs oracle/_ref/libkmc_ref.so, kmc_ref and kmc_tools: `make -C oracle ref cli REF=<KMC source tree>`, then
`python tests/golden/make_reference_digests.py`.  `--only GROUP[,GROUP...]` recomputes only those groups and keeps every other stored
entry (the large bins alone keep the reference busy for a long time); the groups are the keys of GROUPS.
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from kmc_testlib import Params, Reference, bin_digest, result_digest, digest, REFERENCE_DIGESTS  # noqa: E402
import test_oracle_vs_reference as T  # noqa: E402
from test_gpu_parity import LARGE_BINS, large_bin  # noqa: E402


def bins(R, one, out):
    for k, both, cmin in T.BIN_CASES:
        p, b = T.bin_case(k, both, cmin)
        one("bin_k%d_both%d_ci%d" % (k, both, cmin), b, p, T.REF_VARIANTS)
    for cmin, cmax, cntmax in T.CUTOFF_CASES:
        p, b = T.cutoff_case(cmin, cmax, cntmax)
        one("cutoff_ci%d_cx%d_cs%d" % (cmin, cmax, cntmax), b, p, {"raduls": {}})
    for case in sorted(T.CORNER_CASES):
        p, b = T.corner_case(case)
        one(case, b, p, {"raduls": {}})
    for i, b in enumerate(T.edge_bins()):
        one("edge_%d" % i, b, Params(k=31, cutoff_min=1, lut_prefix_len=7), {"raduls": {}})
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    several = T.several_bins()
    res, _ = R.process_bins(several, p, n_sorters=3)
    for i, (b, r) in enumerate(zip(several, res)):
        out["several_%d" % i] = {"input": bin_digest(b), "results": {"raduls_3_sorters": result_digest(r)}}
    for words, key_bytes in T.SORT_CASES:
        recs = T.sort_case(words, key_bytes)
        srt, _ = R.sort(recs, key_bytes, n_threads=2)
        out["sort_w%d_kb%d" % (words, key_bytes)] = {"input": digest(recs), "results": {"raduls_2_threads": digest(srt)}}


def every_k(R, one, out):
    import test_oracle_every_k as E
    for k in E.EVERY_K:
        for both in (True, False):
            p, b = E.every_k_case(k, both)
            one(E.case_name(k, both), b, p, {"raduls": {}})


def databases(R, one, out):
    from kmc_testlib import Oracle
    from test_db_writer import _standalone_bins, write_standalone, db_digest, _expected_dump
    from test_gpu_kmc_files import KMC_TOOLS
    p = Params(k=31, cutoff_min=2, lut_prefix_len=7)
    for case, bins_ in (("standalone_db", _standalone_bins()), ("standalone_db_x3", _standalone_bins() * 3)):
        res = [Oracle().process_bin(b, p) for b in bins_]
        with tempfile.TemporaryDirectory() as tmp:
            db, txt = os.path.join(tmp, "db"), os.path.join(tmp, "dump.txt")
            write_standalone(db, res, p)
            subprocess.check_call([KMC_TOOLS, "transform", db, "dump", txt], stdout=subprocess.DEVNULL)
            assert open(txt).read().split("\n")[:-1] == _expected_dump(res, p), case
            out[case] = {"input": digest(*[bin_digest(b).encode() for b in bins_]), "results": {"kmc_tools_read_back": db_digest(db)}}
    from test_db_writer import REFDB_CASES, REFDB_STATS
    from test_gpu_kmc_files import KMC_REF, write_fastq, count
    import numpy as np
    for k, extra in REFDB_CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            fq = os.path.join(tmp, "reads.fq")
            write_fastq(fq, 500 + k, 200, genome_len=2000, err=0.002)
            db, stats = count(KMC_REF, tmp, "ref", fq, k, extra + ("-sr1", "-n64"))
            np.savez_compressed(os.path.join(HERE, "refdb_k%d.npz" % k), stats=np.array([stats["Stats"][s] for s in REFDB_STATS], dtype=np.int64),
                                **{ext: np.fromfile(db + "." + ext, dtype=np.uint8) for ext in ("kmc_pre", "kmc_suf")})
    import test_reference_cli as CLI
    from test_gpu_kmc_files import dump_sorted
    for k in CLI.CLI_KS:
        with tempfile.TemporaryDirectory() as tmp:
            fq = os.path.join(tmp, "reads.fq")
            CLI.small_fastq(fq)
            db, stats = count(KMC_REF, tmp, "ref", fq, k, ("-ci2", "-cs255"))
            got = {km: int(c) for km, c in (l.split() for l in dump_sorted(tmp, db, "ref").splitlines())}
            out["cli_fastq_k%d" % k] = {"input": digest(open(fq, "rb").read()),
                                        "results": {"dump": CLI.dump_digest(got), "unique_counted_kmers": int(stats["Stats"]["#Unique_counted_k-mers"])}}


def large(R, one, out):
    for case in LARGE_BINS:
        p, b = large_bin(case)
        one(case, b, p, {"raduls": dict(n_sorters=os.cpu_count() or 8)})


GROUPS = {"bins": bins, "every_k": every_k, "databases": databases, "large": large}


def main():
    only = None
    if "--only" in sys.argv:
        only = sys.argv[sys.argv.index("--only") + 1].split(",")
        assert set(only) <= set(GROUPS), "groups: %s" % ", ".join(GROUPS)
    R = Reference()
    out = {}
    if only is not None:
        with open(REFERENCE_DIGESTS) as f:
            out = json.load(f)

    def one(case, b, p, variants):
        res = {name: result_digest(R.process_bin(b, p, **kw)) for name, kw in variants.items()}
        out[case] = {"input": bin_digest(b), "results": res}
        print(case, res[next(iter(res))]["stats"])

    for name, fn in GROUPS.items():
        if only is None or name in only:
            fn(R, one, out)
    with open(REFERENCE_DIGESTS, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
