"""KMC database input (`kmc -fkmc`): the seeded reads the input databases are counted from, the input databases themselves (written by the
reference CLI, kept in tests/golden/kmc_input_dbs.npz), and the cases: what the reference makes of them with `-fkmc -sr1`, kept in
tests/golden/kmc_input_reference.json (tests/golden/make_kmc_input_reference.py writes both)."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KMC_INPUT_DBS = os.path.join(GOLDEN, "kmc_input_dbs.npz")
KMC_INPUT_GOLDEN = os.path.join(GOLDEN, "kmc_input_reference.json")


def write_reads(path, seed, n_reads, read_len, genome_len=1500, err=0.01):
    """A FASTQ of n_reads reads sampled from a random genome (both strands), with substitution errors: repeated and unique k-mers."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    genome = rng.integers(0, 4, genome_len)
    with open(path, "wb") as f:
        for i in range(n_reads):
            at = int(rng.integers(0, genome_len - read_len))
            r = genome[at:at + read_len].copy()
            if rng.random() < 0.5:
                r = 3 - r[::-1]
            e = rng.random(read_len) < err
            r[e] = (r[e] + rng.integers(1, 4, int(e.sum()))) % 4
            f.write(b"@r%d\n%s\n+\n%s\n" % (i, acgt[r].tobytes(), b"I" * read_len))


# The input databases are kept small: few reads, and on the bin path a signature length of 5 and 64 bins, so that the signature map and
# the LUT of every KMC2 .kmc_pre are a few KB.  A run on KMC2 input must use the database's -p and -n (BIN), as in kmc.
BIN = ("-p5", "-n64")

# input database -> (reads seed, reads, read length, k, options of the `kmc` run that writes it)
INPUT_DBS = {
    "k25": (1, 60, 80, 25, ("-ci1",) + BIN),
    "k31": (2, 60, 80, 31, ("-ci1",) + BIN),
    "k32": (4, 40, 80, 32, ("-ci1",) + BIN),
    "k55": (5, 30, 100, 55, ("-ci1",) + BIN),
    "k64": (6, 30, 100, 64, ("-ci1",) + BIN),
    "k128": (7, 16, 160, 128, ("-ci1",) + BIN),
    "k10_kmc1": (8, 60, 80, 10, ("-ci1",)),                             # k <= 13: the small-k path writes KMC1
    "k31_ci5_cs3": (9, 150, 80, 31, ("-ci5", "-cs3") + BIN),           # every stored counter is 3, below its own ci: nothing is read
    "k31_cs1": (10, 30, 80, 31, ("-ci1", "-cs1") + BIN),                # counter_size 0: every record is read
    "k31_cs2": (11, 60, 80, 31, ("-ci2", "-cs1000") + BIN),             # 2-byte counters, min_count 2
    "k31_cs3": (12, 30, 80, 31, ("-ci1", "-cx100000", "-cs100000000") + BIN),   # 3-byte counters, max_count 100000
    "k31_cs4": (13, 30, 80, 31, ("-ci1", "-cs100000000") + BIN),        # 4-byte counters
}

# case -> (input databases, k, options of the `kmc -fkmc` run); the small-k path for k <= 13, as kmc takes it
CASES = {
    "k25_to_k21": (("k25",), 21, ("-ci1",) + BIN),
    "k31_to_k25": (("k31",), 25, ("-ci1",) + BIN),
    "k31_same_k": (("k31",), 31, BIN),
    "k31_to_k33": (("k31",), 33, ("-ci1",) + BIN),                      # every read shorter than k: 0 k-mers
    "k31_to_k11": (("k31",), 11, ("-ci1",)),                            # KMC2 in, small k
    "k32_to_k27": (("k32",), 27, ("-ci1",) + BIN),
    "k55_to_k41": (("k55",), 41, ("-ci1",) + BIN),
    "k64_to_k45": (("k64",), 45, ("-ci1",) + BIN),
    "k128_to_k99": (("k128",), 99, ("-ci1",) + BIN),
    "k128_same_k": (("k128",), 128, ("-ci1",) + BIN),
    "kmc1_k10_to_k9": (("k10_kmc1",), 9, ()),                            # the reference's CI case
    "kmc1_k10_to_k5": (("k10_kmc1",), 5, ("-ci1",)),
    "ci5_cs3_filtered": (("k31_ci5_cs3",), 25, ("-ci1",) + BIN),
    "cs1_no_counters": (("k31_cs1",), 27, ("-ci1",) + BIN),
    "cs2": (("k31_cs2",), 25, ("-ci1",) + BIN),
    "cs3": (("k31_cs3",), 25, ("-ci1",) + BIN),
    "cs4": (("k31_cs4",), 25, ("-ci1",) + BIN),
    "both_strands_off": (("k31",), 25, ("-ci1", "-b") + BIN),
    "hc": (("k31",), 21, ("-ci1", "-hc") + BIN),
    "opt_out_size": (("k31",), 25, ("-ci1", "--opt-out-size") + BIN),
    "two_dbs": (("k31", "k25"), 21, ("-ci1",) + BIN),                    # the map comes from the first
    "estimate": (("k31",), 21, ("-e",)),
}

# refusal -> (input database, k, options, the reference's message)
REFUSALS = {
    "kmc1_on_bin_path": ("k10_kmc1", 25, BIN, "currently only KMC databases in version 2 can be readed. If needed to read other version "
                         "please post an GitHub issue."),
    "signature_len": ("k31", 25, ("-p7", "-n64"), "Wrong signature length, should be the same as input KMC database: 5"),
    "n_bins": ("k31", 25, ("-p5", "-n256"), "Wrong number of bins, should be the same as input KMC database: 64"),
}


def options(opts):
    """count_reads / count_reads_small_k / estimate_histogram keywords of a case's kmc options."""
    kw = {"cutoff_min": 2, "cutoff_max": 1_000_000_000, "counter_max": 255, "both_strands": True, "homopolymer_compressed": False,
          "opt_out_size": False, "n_bins": None, "signature_len": 9}
    for o in opts:
        if o.startswith("-ci"):
            kw["cutoff_min"] = int(o[3:])
        elif o.startswith("-cx"):
            kw["cutoff_max"] = int(o[3:])
        elif o.startswith("-cs"):
            kw["counter_max"] = int(o[3:])
        elif o == "-b":
            kw["both_strands"] = False
        elif o == "-hc":
            kw["homopolymer_compressed"] = True
        elif o == "--opt-out-size":
            kw["opt_out_size"] = True
        elif o.startswith("-p"):
            kw["signature_len"] = int(o[2:])
        elif o.startswith("-n"):
            kw["n_bins"] = int(o[2:])
    return kw


def materialize(tmp, names=None):
    """Writes the input databases (all, or `names`) from tests/golden/kmc_input_dbs.npz under tmp; returns {name: prefix}."""
    z = np.load(KMC_INPUT_DBS)
    out = {}
    for name in names or INPUT_DBS:
        prefix = os.path.join(str(tmp), "in_" + name)
        for ext in ("kmc_pre", "kmc_suf"):
            z["%s.%s" % (name, ext)].tofile(prefix + "." + ext)
        out[name] = prefix
    return out
