"""Stores what the unmodified reference CLI writes in its small-k mode (k <= 13) for test_small_k_model.CASES:
tests/golden/small_k_reference.json, per case the kmc arguments, the MD5 of the generated input and of both database files, the .kmc_pre
footer fields and the totals of `-j`.

Every run is checked to have taken the small-k path: only CSmallKCompleter writes the KMC1 format (version word 0 in .kmc_pre); with too
little -m the reference falls back to bins silently, so the memory given here leaves room for the 4^13 counters.

Needs oracle/_ref/kmc_ref (`make -C oracle cli REF=<KMC source tree>`), then `python tests/golden/make_small_k_reference.py`.
"""
import hashlib
import json
import os
import struct
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from test_small_k_model import CASES, GOLDEN, kmc_args, write_input  # noqa: E402
from test_gpu_kmc_files import KMC_REF  # noqa: E402


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def footer(pre_path):
    pre = open(pre_path, "rb").read()
    version, offset = struct.unpack("<II", pre[-12:-4])
    f = pre[-8 - offset:-8]
    k, mode, cs, lp, cmin, cmax_lo, n = struct.unpack("<IIIIIIQ", f[:32])
    return {"version": version, "kmer_len": k, "mode": mode, "counter_size": cs, "lut_prefix_len": lp, "cutoff_min": cmin,
            "cutoff_max_lo": cmax_lo, "n_counted": n, "both_strands": f[32] == 0, "cutoff_max_hi": struct.unpack("<I", f[36:40])[0]}


def run_case(case, tmp, binary=KMC_REF):
    """Runs the reference on the case's input; returns the stored entry and the database prefix."""
    inp = os.path.join(tmp, "input")
    write_input(case, inp)
    db, wd, js = os.path.join(tmp, "db"), os.path.join(tmp, "wd"), os.path.join(tmp, "stats.json")
    os.makedirs(wd, exist_ok=True)
    subprocess.run([binary] + kmc_args(case) + ["-m4", "-t4", "-j" + js, inp, db, wd], check=True, stdout=subprocess.DEVNULL,
                   stderr=subprocess.DEVNULL)
    st = json.load(open(js))["Stats"]
    ent = {"args": kmc_args(case), "input_md5": md5(inp), "kmc_pre_md5": md5(db + ".kmc_pre"), "kmc_suf_md5": md5(db + ".kmc_suf")}
    ent.update(footer(db + ".kmc_pre"))
    ent.update({"n_unique": int(st["#Unique_k-mers"]), "n_cutoff_min": int(st["#k-mers_below_min_threshold"]),
                "n_cutoff_max": int(st["#k-mers_above_max_threshold"]), "n_total": int(st["#Total no. of k-mers"])})
    assert ent["version"] == 0, "%s: the reference did not take its small-k path (version %d)" % (case[0], ent["version"])
    assert ent["n_counted"] == int(st["#Unique_counted_k-mers"])
    return ent, db


def main():
    out = {}
    for case in CASES:
        with tempfile.TemporaryDirectory() as tmp:
            out[case[0]], _ = run_case(case, tmp)
        print(case[0], out[case[0]]["lut_prefix_len"], out[case[0]]["n_counted"])
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
