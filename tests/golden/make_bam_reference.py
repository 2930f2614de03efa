"""Stores what the unmodified reference CLI makes of a BAM file (tests/bam_testlib.BAM_CASES) with `-fbam -sr1`, so that the tests run
without a reference build: tests/golden/bam_reference.json.  Per case the MD5 of the decompressed BAM (the compressed bytes depend on the
zlib build), the MD5 of kmc_b200.reads.bam_to_batch's batch, and the MD5s of .kmc_pre / .kmc_suf with the -j totals, or of the -e file.

The script asserts that every member layout of the same records gives the reference the same files, and that the reference writes the
same files for a multi-FASTA of the model's batch (`-fm`): together these pin the model to the reference's own BAM reader.

Needs oracle/_ref/kmc_ref (`make -C oracle cli REF=<KMC source tree>`), then `python tests/golden/make_bam_reference.py`.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from bam_testlib import BAM_CASES, BAM_GOLDEN, LAYOUTS, case_bam  # noqa: E402
from gzip_testlib import write  # noqa: E402
from kmc_b200.reads import bam_to_batch  # noqa: E402
from test_gpu_kmc_files import KMC_REF, count  # noqa: E402


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def reference(tmp, tag, path, fmt, k, opts):
    if "-e" in opts:
        out = os.path.join(tmp, "hist_%s.txt" % tag)
        subprocess.run([KMC_REF, "-k%d" % k, fmt, "-t4", "-m2"] + opts + [path, out, tmp], check=True, stdout=subprocess.DEVNULL,
                       stderr=subprocess.DEVNULL)
        return {"histogram_md5": md5(out)}
    db, stats = count(KMC_REF, tmp, tag, path, k, tuple(opts) + ("-sr1",), fmt=fmt)
    st = stats.get("Stats", stats)
    return {"kmc_pre_md5": md5(db + ".kmc_pre"), "kmc_suf_md5": md5(db + ".kmc_suf"), "total_kmers": int(st["#Total no. of k-mers"]),
            "unique_kmers": int(st["#Unique_k-mers"]), "counted_kmers": int(st["#Unique_counted_k-mers"])}


def multi_fasta(batch):
    lines = bytes(batch).split(b"\n")[:-1]
    return b"".join(b">r\n%s\n" % s for s in lines)


def main():
    cases = {}
    with tempfile.TemporaryDirectory() as tmp:
        files = {}
        for layout in LAYOUTS:
            raw, text = case_bam(layout)
            files[layout] = write(os.path.join(tmp, "in_%s.bam" % layout), raw)
        for name, (k, opts, _) in BAM_CASES.items():
            original = "-b" in opts
            batch = bam_to_batch(text, original_strand=original)
            ent = reference(tmp, name + "_aligned", files["aligned"], "-fbam", k, opts)
            for layout in LAYOUTS[1:]:
                assert ent == reference(tmp, name + "_" + layout, files[layout], "-fbam", k, opts), "%s: layout %s differs" % (name, layout)
            fa = write(os.path.join(tmp, name + ".fa"), multi_fasta(batch))
            assert ent == reference(tmp, name + "_fm", fa, "-fm", k, opts), "%s: the reference wrote other files for the model's batch" % name
            ent.update({"options": opts, "k": k, "bam_md5": hashlib.md5(text).hexdigest(), "batch_md5": hashlib.md5(batch.tobytes()).hexdigest()})
            cases[name] = ent
            print(name, ent)
    with open(BAM_GOLDEN, "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
