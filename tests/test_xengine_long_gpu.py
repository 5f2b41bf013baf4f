"""GPU: the device engine (bt2g_xengine_*) on reads of 300 to 512 bases, 2 x 300 bp pairs and mate windows up to 8000 columns, against
the reference program run here (--seed 0 --reorder): every SAM record identical.

Under default end-to-end scoring an engine whose longest read passes about 210 bases sends every DP through the s16x2 move-code
kernel; reads of 424 bases and more take the reference's i16 matrix end-to-end (another reseed per backtrace than the u8 one); a
--score-min that keeps the range in a byte puts 450 bp reads on the split H-byte kernels at 16 rows per lane; -X 5000 and -X 7600
make mate windows of about 5400 and 7800 columns in the device engine; -X 8000 windows (about 8200 columns) pass its 8000-column mate
workspace and are finished by the coroutine engine."""
import subprocess

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from bowtie2_b200 import Bt2Gpu
    return Bt2Gpu(0)


@pytest.fixture(scope="module")
def genomes(tmp_path_factory):
    """the repeat-rich genome of test_xengine_gpu (.bt2 and .bt2l), and one of two 60 kbp contigs for inserts of 1-5 kbp"""
    from bowtie2_b200 import synth
    from oracle_lib import have_reference, ref_bin
    if not have_reference():
        pytest.skip("oracle/_ref not built")
    d = tmp_path_factory.mktemp("xlong")
    out = {}
    for name, g, builders in [("rep", synth.make_genome(n_contigs=3, contig_len=200000, seed=17, repeat_frac=0.2, repeat_len=400,
                                                        repeat_copies=150, n_gap=53), ("s", "l")),
                              ("wide", synth.make_genome(n_contigs=2, contig_len=60000, seed=23, repeat_frac=0.05, repeat_len=300,
                                                         repeat_copies=10, n_gap=40), ("s",))]:
        fa = str(d / (name + ".fa"))
        synth.write_fasta(fa, g)
        for b in builders:
            subprocess.check_call([ref_bin("bowtie2-build-" + b), "--seed", "0", "--quiet", fa, str(d / (name + b))])
        out[name] = (g, str(d / name))
    return out


def _long_pairs(genome, n, L, seed, frag_lo, frag_hi):
    """FR pairs with fragments of frag_lo..frag_hi bases (synth.make_pairs caps them at 500): mate 1 the fragment's left end on a
    random strand, mate 2 the reverse complement of its right end, 1% substitutions"""
    from bowtie2_b200 import synth
    rng = np.random.default_rng(seed)
    reads, quals = [], []
    for _ in range(n):
        c = int(rng.integers(0, len(genome)))
        f = int(rng.integers(frag_lo, frag_hi + 1))
        p = int(rng.integers(0, len(genome[c]) - f))
        frag = genome[c][p:p + f].copy()
        frag[frag > 3] = 0
        if rng.integers(0, 2):
            frag = synth.revcomp(frag)
        m1, m2 = frag[:L].copy(), synth.revcomp(frag[-L:])
        for m in (m1, m2):
            k = rng.random(L) < 0.01
            m[k] = (m[k] + 1 + rng.integers(0, 3, int(k.sum()))) % 4
            reads.append(m.astype(np.uint8))
            quals.append(rng.integers(35, 74, L).astype(np.uint8))
    return reads, quals


CASES = {
    # name: (genome, index suffix, paired, local, preset, read length, units, reference arguments, engine keyword arguments)
    "U300": ("rep", "s", False, False, "sensitive", 300, 800, [], {}),
    "U512": ("rep", "s", False, False, "sensitive", 512, 600, [], {}),
    "U-ragged-100-512": ("rep", "s", False, False, "sensitive", "ragged", 800, [], {}),
    "P300-vs": ("rep", "s", True, False, "very-sensitive", 300, 600, [], {}),
    "P300-vs-X1000": ("rep", "s", True, False, "very-sensitive", 300, 600, ["-X", "1000"], {"maxfrag": 1000}),
    "P300-bt2l": ("rep", "l", True, False, "sensitive", 300, 500, [], {}),
    "P300-k3": ("rep", "s", True, False, "sensitive", 300, 400, ["-k", "3"], {"k": 3}),
    "P250-local": ("rep", "s", True, True, "sensitive", 250, 600, [], {}),
    "U400-vs-local": ("rep", "s", False, True, "very-sensitive", 400, 500, [], {}),
    "U450-score-min": ("rep", "s", False, False, "sensitive", 450, 600, ["--score-min", "L,0,-0.2"], {"score_min": (0.0, -0.2)}),
    "P150-X5000": ("wide", "s", True, False, "sensitive", 150, 600, ["-X", "5000"], {"maxfrag": 5000}),
    "P150-X7600": ("wide", "s", True, False, "sensitive", 150, 600, ["-X", "7600"], {"maxfrag": 7600}),
    "P150-X8000": ("wide", "s", True, False, "sensitive", 150, 600, ["-X", "8000"], {"maxfrag": 8000}),
}
# units the coroutine engine may finish per case: the counts observed on an H100 (in the comments) plus about a quarter.  Long reads
# overflow the device engine's per-unit capacities far more often than 100-250 bp reads do
_MAX_FALLBACK = {
    "U300": 60,                 # 48 of 800
    "U512": 145,                # 114 of 600
    "U-ragged-100-512": 75,     # 59 of 800
    "P300-vs": 165,             # 132 of 600
    "P300-vs-X1000": 165,       # 132 of 600
    "P300-bt2l": 40,            # 30 of 500
    "P300-k3": 115,             # 90 of 400
    "P250-local": 105,          # 83 of 600
    "U400-vs-local": 145,       # 114 of 500
    "U450-score-min": 135,      # 107 of 600
    "P150-X5000": 10,           # 0 of 600
    "P150-X7600": 10,
    # 553 of 600: mate windows of -X 8000 (about 8200 columns) pass the device engine's 8000-column mate workspace, so their units
    # are finished by the coroutine engine (bt2g_dp_extend, which takes windows up to 16384 columns)
    "P150-X8000": 600,
}


def _reads(genome, paired, local, L, n, seed, wide):
    from bowtie2_b200 import synth
    if wide:
        return _long_pairs(genome, n, L, seed, 1000, 5000)
    if paired:
        reads, quals, _ = synth.make_pairs(genome, n, L, seed=seed, sub_rate=0.01, indel_rate=0.001, ins_mean=420, ins_sd=60)
        return reads, quals
    if L == "ragged":
        reads, quals, _ = synth.make_reads(genome, n, 512, seed=seed, sub_rate=0.01, indel_rate=0.001)
        rng = np.random.default_rng(seed)
        cut = [512] + [int(x) for x in rng.integers(100, 513, n - 1)]        # one read of 512: the engine's maxLen
        return [r[:k] for r, k in zip(reads, cut)], [q[:k] for q, k in zip(quals, cut)]
    reads, quals, _ = synth.make_reads(genome, n, L, seed=seed, sub_rate=0.01, indel_rate=0.001)
    return reads, quals


@pytest.mark.parametrize("case", list(CASES))
def test_long_reads_device_engine_equals_the_reference_program(genomes, tmp_path, case):
    from bowtie2_b200 import policy, synth
    from bowtie2_b200.lib import ReadBatch, XEngine, load_library, policy_params, sam_format
    from oracle_lib import ref_bin
    gname, sfx, paired, local, preset, L, n, args, kw = CASES[case]
    genome, base = genomes[gname]
    base += sfx
    reads, quals = _reads(genome, paired, local, L, n, 43 + n, gname == "wide")
    if paired:
        f1, f2 = str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")
        synth.write_fastq(f1, reads[0::2], quals[0::2]); synth.write_fastq(f2, reads[1::2], quals[1::2])
        io = ["-1", f1, "-2", f2]
    else:
        fq = str(tmp_path / "r.fq")
        synth.write_fastq(fq, reads, quals)
        io = ["-U", fq]
    names = [f"r{i // 2}" for i in range(2 * n)] if paired else [f"r{i}" for i in range(n)]
    out = subprocess.check_output([ref_bin("bowtie2-align-" + sfx), *(["--local"] if local else []), "--" + preset + ("-local" if local else ""),
                                   *args, "--seed", "0", "-p", "4", "--reorder", "-x", base] + io, stderr=subprocess.DEVNULL).decode()
    want = [l for l in out.split("\n") if l and not l.startswith("@")]
    ref_names = [l.split("\t")[1][3:] for l in out.split("\n") if l.startswith("@SQ")]
    pkw = {}
    if "maxfrag" in kw:
        pkw["pe"] = policy.PairedEndPolicy(local=local, maxfrag=kw["maxfrag"])
    fmt = {}
    if "score_min" in kw:
        sc = policy.Scoring.default(local)
        sc.score_min_func = policy.SimpleFunc(policy.SIMPLE_FUNC_LINEAR, *kw["score_min"])
        pkw["sc"] = fmt["sc"] = sc
    g = _gpu()
    try:
        g.load_index_files(base)
        batch = ReadBatch.from_list(reads, quals)
        if "k" in kw:                                                     # -k: every reported alignment (align_k)
            from bowtie2_b200.align import expand_entries
            eng = XEngine(g, policy_params(preset, local=local, paired=paired, k=kw["k"]), n, max(len(r) for r in reads),
                          max_per_unit=8)                             # (room for the pair entries of -k 3, as in test_xengine_k_gpu)
            try:
                res, ops, pairs, cnt, truncated, stats = eng.align_k(batch, names)
            finally:
                eng.close()
            assert not truncated
            batch, names, res, ops, pairs = expand_entries(batch, names, res, ops, cnt, pairs)
        else:
            eng = XEngine(g, policy_params(preset, local=local, paired=paired, **pkw), n, max(len(r) for r in reads))
            try:
                res, ops, pairs, stats = eng.align(batch, names)
            finally:
                eng.close()
        lines = sam_format(load_library(), batch, res, ops, ref_names, read_names=names, pairs=pairs, local=local, **fmt).rstrip("\n").split("\n")
    finally:
        g.close()
    bad = [i for i in range(len(want)) if lines[i] != want[i]]
    print(f"{case}: {len(want)} records, {stats['fallback_units']} of {n} units finished by the coroutine engine, "
          f"{stats['seed_dps']} seed DPs, {stats.get('mate_dps', 0)} mate DPs")
    assert len(lines) == len(want) and not bad, (len(bad), lines[bad[0]] if bad else None, want[bad[0]] if bad else None, stats)
    assert stats["seed_dps"] > 100, stats
    if paired and not local:
        assert stats["mate_dps"] > 50, stats
    assert stats["fallback_units"] <= _MAX_FALLBACK[case], stats
