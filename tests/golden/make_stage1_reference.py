"""Stores what the unmodified reference CLI makes of the stage-1 test reads (tests/stage1_testlib.STAGE1_CASES), so that the stage-1
tests run without a reference build: tests/golden/stage1_reference.json (database header fields, per file bin the SHA-256 of its
payload slice of .kmc_suf and of its raw LUT counts, digests of the two files, #Total_super-k-mers and #Total no. of k-mers from -j) and
tests/golden/stage1_maps.npz (the signature map stored in each .kmc_pre, uint16).  The reads are regenerated from their seeds.

Needs oracle/_ref/kmc_ref: `make -C oracle cli REF=<KMC source tree>`, then `python tests/golden/make_stage1_reference.py`.
"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from kmc_testlib import digest  # noqa: E402
from stage1_testlib import STAGE1_CASES, STAGE1_GOLDEN, STAGE1_MAPS, case_reads, kmc_pre_bins, write_fastq_reads  # noqa: E402
from test_gpu_kmc_files import KMC_REF, count  # noqa: E402

REF_OPTIONS = ("-sr1", "-n64")


def run_case(tmp, name):
    seed, profile, n_reads, read_len, k, extra = STAGE1_CASES[name]
    fq = os.path.join(tmp, name + ".fq")
    write_fastq_reads(fq, case_reads(name))
    db, stats = count(KMC_REF, tmp, name, fq, k, tuple(extra) + REF_OPTIONS)
    return db, stats


def main():
    cases, maps = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (seed, profile, n_reads, read_len, k, extra) in STAGE1_CASES.items():
            db, stats = run_case(tmp, name)
            header, sig_map, payloads, raw = kmc_pre_bins(db + ".kmc_pre", db + ".kmc_suf")
            st = stats.get("Stats", stats)
            cs = [int(x[3:]) for x in extra if x.startswith("-cs")]
            cases[name] = {
                "header": header, "counter_max": cs[0] if cs else 255, "options": list(extra) + list(REF_OPTIONS),
                "bins": [{"payload": digest(payloads[b]), "lut": digest(raw[b])} for b in range(raw.shape[0])],
                "files": {ext: digest(open(db + ext, "rb").read()) for ext in (".kmc_pre", ".kmc_suf")},
                "total_super_kmers": int(st["#Total_super-k-mers"]) if "#Total_super-k-mers" in st else None,
                "total_kmers": int(st["#Total no. of k-mers"]),
            }
            maps[name] = sig_map.astype(np.uint16)
            print(name, header, cases[name]["total_kmers"], cases[name]["total_super_kmers"])
    np.savez_compressed(STAGE1_MAPS, **maps)
    with open(STAGE1_GOLDEN, "w") as f:
        json.dump({"cases": cases}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
