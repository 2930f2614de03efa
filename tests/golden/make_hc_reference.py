"""Stores what the unmodified reference CLI makes of the homopolymer-compression cases (tests/hc_testlib.HC_CASES) with `-hc -sr1`, so that
the tests run without a reference build: tests/golden/hc_reference.json and tests/golden/hc_maps.npz (the signature map of every bin-path
case's .kmc_pre, uint16).  Per case:
  bin path  the database header, per file bin the digests of its payload slice of .kmc_suf and of its raw LUT counts, the MD5s of the two
            files, and #Total no. of k-mers, #Total_super-k-mers and #Unique_k-mers from -j;
  small k   the MD5s of the two files, the KMC1 footer (version word 0: the reference took its small-k path) and the -j totals;
  -e        the MD5 of the histogram file; the script checks that `kmc -e -hc` writes the file `kmc -e` writes.
The reads are regenerated from their seeds; the MD5 of each input is stored with it.

Needs oracle/_ref/kmc_ref (`make -C oracle cli REF=<KMC source tree>`), then `python tests/golden/make_hc_reference.py`.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from hc_testlib import HC_CASES, HC_GOLDEN, HC_MAPS, case_format, case_options, option, write_case_input  # noqa: E402
from kmc_testlib import digest  # noqa: E402
from make_small_k_reference import footer  # noqa: E402
from stage1_testlib import kmc_pre_bins  # noqa: E402
from test_gpu_kmc_files import KMC_REF, count  # noqa: E402

REF_OPTIONS = ("-hc", "-sr1")


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def histogram_file(tmp, tag, path, name, hc):
    out = os.path.join(tmp, "hist_%s.txt" % tag)
    cmd = [KMC_REF, "-k%d" % HC_CASES[name][4], case_format(name), "-t4", "-m2", "-e"] + (["-hc"] if hc else []) + [path, out, tmp]
    subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return md5(out)


def run_case(tmp, name):
    k = HC_CASES[name][4]
    path = os.path.join(tmp, name + ".input")
    write_case_input(name, path)
    ent = {"options": case_options(name) + [case_format(name)] + list(REF_OPTIONS), "input_md5": md5(path)}
    if "-e" in HC_CASES[name][5]:
        ent["options"] = case_options(name) + [case_format(name), "-hc"]
        ent["histogram_md5"] = histogram_file(tmp, name + "_hc", path, name, True)
        assert ent["histogram_md5"] == histogram_file(tmp, name, path, name, False), "%s: kmc -e -hc wrote another file than kmc -e" % name
        return ent, None
    db, stats = count(KMC_REF, tmp, name, path, k, tuple(case_options(name)) + REF_OPTIONS, fmt=case_format(name))
    st = stats.get("Stats", stats)
    ent.update({"kmc_pre_md5": md5(db + ".kmc_pre"), "kmc_suf_md5": md5(db + ".kmc_suf"), "total_kmers": int(st["#Total no. of k-mers"]),
                "unique_kmers": int(st["#Unique_k-mers"]), "counted_kmers": int(st["#Unique_counted_k-mers"])})
    if k <= 13:
        ent.update(footer(db + ".kmc_pre"))
        assert ent["version"] == 0, "%s: the reference did not take its small-k path" % name
        return ent, None
    header, sig_map, payloads, raw = kmc_pre_bins(db + ".kmc_pre", db + ".kmc_suf")
    ent.update({"header": header, "counter_max": option(name, "-cs", 255), "total_super_kmers": int(st["#Total_super-k-mers"]),
                "bins": [{"payload": digest(payloads[b]), "lut": digest(raw[b])} for b in range(raw.shape[0])]})
    return ent, sig_map.astype(np.uint16)


def main():
    cases, maps = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for name in HC_CASES:
            cases[name], sig_map = run_case(tmp, name)
            if sig_map is not None:
                maps[name] = sig_map
            print(name, {key: v for key, v in cases[name].items() if key not in ("bins",)})
    np.savez_compressed(HC_MAPS, **maps)
    with open(HC_GOLDEN, "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
