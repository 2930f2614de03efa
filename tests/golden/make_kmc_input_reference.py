"""Stores what the unmodified reference CLI makes of KMC databases with `-fkmc -sr1` (tests/kmc_input_testlib.CASES), so that the tests
run without a reference build: the reference-written input databases go to tests/golden/kmc_input_dbs.npz, and per case the MD5s of the
output .kmc_pre / .kmc_suf with the -j totals (or the MD5 of the -e file), plus the MD5 of kmc_b200.reads.kmc_db_to_batch's batch, go to
tests/golden/kmc_input_reference.json with the messages of the three refusals.

The script asserts that the model is the reference's reader: on the small-k path, `-fa` on the model's batch written as FASTA
(">\\n<k-mer>\\n" per record, what CBinaryFilesReader::ProcessKMC prints) gives the same files as `-fkmc`; on the bin path, where the signature
map of `-fa` comes from stage 0 instead of the input database, `kmc_tools transform ... dump -s` of both outputs is the same listing.

Needs oracle/_ref/kmc_ref and kmc_tools (`make -C oracle cli REF=<KMC source tree>`), then `python tests/golden/make_kmc_input_reference.py`.
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

from kmc_input_testlib import CASES, INPUT_DBS, KMC_INPUT_DBS, KMC_INPUT_GOLDEN, REFUSALS, write_reads  # noqa: E402
from kmc_b200.reads import kmc_db_to_batch  # noqa: E402
from test_gpu_kmc_files import KMC_REF, KMC_TOOLS  # noqa: E402


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def kmc(tmp, inputs, out, k, opts, fmt="-fkmc", check=True):
    wd = tempfile.mkdtemp(dir=tmp)
    js = out + ".json"
    cmd = [KMC_REF, "-k%d" % k, fmt, "-t4", "-m2", "-j" + js] + list(opts)
    if len(inputs) > 1:
        lst = out + ".lst"
        open(lst, "w").write("".join(p + "\n" for p in inputs))
        cmd += ["@" + lst, out, wd]
    else:
        cmd += [inputs[0], out, wd]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    if check and r.returncode:
        raise RuntimeError("%s failed: %s" % (" ".join(cmd), r.stderr))
    return r, (json.load(open(js)) if r.returncode == 0 and os.path.exists(js) and "-e" not in opts else None)


def dump(tmp, db):
    txt = db + ".dump"
    subprocess.run([KMC_TOOLS, "transform", db, "dump", "-s", txt], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return open(txt).read()


def main():
    cases, dbs = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        prefix = {}
        for name, (seed, n_reads, read_len, k, opts) in INPUT_DBS.items():
            fq = os.path.join(tmp, "reads_%s.fq" % name)
            write_reads(fq, seed, n_reads, read_len)
            prefix[name] = os.path.join(tmp, "in_" + name)
            kmc(tmp, [fq], prefix[name], k, opts, fmt="-fq")
            for ext in ("kmc_pre", "kmc_suf"):
                dbs["%s.%s" % (name, ext)] = np.fromfile(prefix[name] + "." + ext, dtype=np.uint8)
        for name, (inputs, k, opts) in CASES.items():
            paths = [prefix[i] for i in inputs]
            batch = np.concatenate([kmc_db_to_batch(p) for p in paths])
            fa = os.path.join(tmp, name + ".fa")
            with open(fa, "wb") as f:
                f.write(b"".join(b">\n" + s + b"\n" for s in batch.tobytes().split(b"\n")[:-1]))
            out = os.path.join(tmp, "out_" + name)
            ent = {"inputs": list(inputs), "k": k, "options": list(opts), "batch_md5": hashlib.md5(batch.tobytes()).hexdigest()}
            if "-e" in opts:
                kmc(tmp, paths, out, k, opts)
                kmc(tmp, [fa], out + "_fa", k, opts, fmt="-fa")
                assert md5(out) == md5(out + "_fa"), "%s: -e differs between -fkmc and the model's FASTA" % name
                ent["histogram_md5"] = md5(out)
            else:
                _, st = kmc(tmp, paths, out, k, list(opts) + ["-sr1"])
                st = st.get("Stats", st)
                ent.update({"kmc_pre_md5": md5(out + ".kmc_pre"), "kmc_suf_md5": md5(out + ".kmc_suf"),
                            "total_kmers": int(st["#Total no. of k-mers"]), "unique_kmers": int(st["#Unique_k-mers"]),
                            "counted_kmers": int(st["#Unique_counted_k-mers"]), "n_reads": int(st["#Total_reads"])})
                _, st_fa = kmc(tmp, [fa], out + "_fa", k, list(opts) + ["-sr1"], fmt="-fa")
                if k <= 13:
                    assert (md5(out + ".kmc_pre"), md5(out + ".kmc_suf")) == (md5(out + "_fa.kmc_pre"), md5(out + "_fa.kmc_suf")), \
                        "%s: the small-k files differ between -fkmc and the model's FASTA" % name
                elif ent["counted_kmers"]:
                    assert dump(tmp, out) == dump(tmp, out + "_fa"), "%s: the listing differs between -fkmc and the model's FASTA" % name
            cases[name] = ent
            print(name, ent)
        refusals = {}
        for name, (inp, k, opts, msg) in REFUSALS.items():
            r, _ = kmc(tmp, [prefix[inp]], os.path.join(tmp, "refused_" + name), k, opts, check=False)
            assert r.returncode != 0 and msg in r.stdout + r.stderr, "%s: %r not in %r" % (name, msg, r.stdout + r.stderr)
            refusals[name] = msg
    np.savez_compressed(KMC_INPUT_DBS, **dbs)
    with open(KMC_INPUT_GOLDEN, "w") as f:
        json.dump({"cases": cases, "refusals": refusals}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
