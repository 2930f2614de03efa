"""Stores what the unmodified reference CLI makes of BGZF-compressed inputs (tests/gzip_testlib.GZIP_CASES) with `-sr1`, so that the tests
run without a reference build: tests/golden/gzip_reference.json.  Per case the MD5 of the decompressed input (the compressed bytes depend on
the zlib build, the text and the databases do not), and the MD5s of .kmc_pre / .kmc_suf with the -j totals, or of the -e file.  The script
also checks that the reference writes the same files for the text uncompressed.

Needs oracle/_ref/kmc_ref (`make -C oracle cli REF=<KMC source tree>`), then `python tests/golden/make_gzip_reference.py`.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from gzip_testlib import FORMAT_FLAG, GZIP_CASES, GZIP_GOLDEN, bgzf, case_text, write  # noqa: E402
from test_gpu_kmc_files import KMC_REF, count  # noqa: E402


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def reference(tmp, tag, path, kind, k, opts):
    if "-e" in opts:
        out = os.path.join(tmp, "hist_%s.txt" % tag)
        subprocess.run([KMC_REF, "-k%d" % k, FORMAT_FLAG[kind], "-t4", "-m2"] + opts + [path, out, tmp], check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        return {"histogram_md5": md5(out)}
    db, stats = count(KMC_REF, tmp, tag, path, k, tuple(opts) + ("-sr1",), fmt=FORMAT_FLAG[kind])
    st = stats.get("Stats", stats)
    return {"kmc_pre_md5": md5(db + ".kmc_pre"), "kmc_suf_md5": md5(db + ".kmc_suf"), "total_kmers": int(st["#Total no. of k-mers"]),
            "unique_kmers": int(st["#Unique_k-mers"]), "counted_kmers": int(st["#Unique_counted_k-mers"])}


def main():
    cases = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (kind, k, opts, _) in GZIP_CASES.items():
            text = case_text(kind)
            plain = write(os.path.join(tmp, name + ".txt"), text)
            gz = write(os.path.join(tmp, name + ".gz"), bgzf(text))
            ent = reference(tmp, name + "_gz", gz, kind, k, opts)
            assert ent == reference(tmp, name, plain, kind, k, opts), "%s: the reference wrote other files for the plain text" % name
            ent.update({"options": opts, "k": k, "input": kind, "text_md5": hashlib.md5(text).hexdigest()})
            cases[name] = ent
            print(name, ent)
    with open(GZIP_GOLDEN, "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
