"""SeedAligner::oneMmSearch: C restatement vs reference (CPU) and CUDA vs restatement (GPU)."""
import numpy as np
import pytest

from bowtie2_b200 import synth
import oracle_lib
from oracle_lib import Oracle, Reference, have_reference, oracle_one_mm, ref_one_mm, scoring_grid

# the scorings of oracle_lib.scoring_grid() that the 1-mismatch search reads: mismatch and N penalties, the match bonus
GRID = ["mp6,6", "mp2,2", "mp8,3", "np0", "np3", "local-ma1", "local-ma3"]


def _cases(genome, seed=33):
    """Reads of mixed length with 0, 1 or 2 substitutions, some Ns, random qualities."""
    rng = np.random.default_rng(seed)
    out = []
    for ln, n in ((12, 30), (15, 30), (19, 30), (20, 20), (21, 20), (33, 30), (64, 30), (101, 40), (250, 10)):
        reads, _, _ = synth.make_reads(genome, n, ln, seed=seed + ln, sub_rate=0.0, indel_rate=0.0)
        for k, r in enumerate(reads):
            nsub = (1, 1, 1, 0, 2, 1)[k % 6]
            for p in rng.choice(ln, size=nsub, replace=False):
                r[p] = (r[p] + rng.integers(1, 4)) % 4
            if k % 7 == 3:
                r[rng.integers(0, ln)] = 4
            if k % 29 == 11:
                r[rng.integers(0, ln)] = 4
            q = rng.integers(33, 74, size=ln).astype(np.uint8)
            out.append((r.astype(np.uint8), q))
    return out


def _minsc(ln, local, k):
    if local:
        return (int(20 + 8.0 * np.log(ln)), 2 * ln - 3, 1)[k % 3]
    return (int(-0.6 - 0.6 * ln), -3, -6)[k % 3]


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("local", [False, True])
def test_onemm_oracle_vs_reference(local, synth_index, synth_genome):
    assert _oracle_vs_reference(Oracle(synth_index), Reference(synth_index), local, synth_genome) > 50


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", GRID)
def test_onemm_oracle_vs_reference_under_scoring(name, synth_index, synth_genome):
    sc = scoring_grid()[name]
    O, R = Oracle(synth_index), Reference(synth_index)
    R.set_scoring(sc)
    oracle_lib.SCORING_OVERRIDE = sc
    try:
        assert _oracle_vs_reference(O, R, sc.local, synth_genome) > 50
    finally:
        oracle_lib.SCORING_OVERRIDE = None


def _oracle_vs_reference(O, R, local, genome):
    nhit = 0
    for k, (r, q) in enumerate(_cases(genome)):
        minsc = _minsc(len(r), local, k)
        nofw, norc = (k % 11 == 5), (k % 13 == 7)
        a = oracle_one_mm(O, local, r, q, minsc, nofw, norc)
        b = ref_one_mm(R, local, r, q, minsc, nofw, norc)
        assert a == b, (k, len(r), a, b)
        nhit += len(a)
    return nhit


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("which,local,scoring", [pytest.param("small", False, None, id="small-False"), pytest.param("small", True, None, id="small-True"),
                                                 pytest.param("large", False, None, id="large-False")] +
                         [pytest.param("small", name.startswith("local"), name, id="small-" + name) for name in ("mp8,3", "mp2,2", "np0", "local-ma3")])
def test_onemm_gpu_vs_oracle(which, local, scoring, gpu, synth_index, synth_index_large, synth_genome):
    """the kernel and the restatement under the default scorings and, as gpu.set_scoring_policy installs them, some of the grid's"""
    base = synth_index if which == "small" else synth_index_large
    gpu.load_index_files(base)
    if scoring is None:
        gpu.set_scoring(local=local)
    else:
        oracle_lib.SCORING_OVERRIDE = scoring_grid()[scoring]
        gpu.set_scoring_policy(oracle_lib.SCORING_OVERRIDE)
    try:
        _gpu_vs_oracle(gpu, Oracle(base), local, synth_genome)
    finally:
        oracle_lib.SCORING_OVERRIDE = None
        gpu.set_scoring(local=False)


def _gpu_vs_oracle(gpu, O, local, synth_genome):
    from bowtie2_b200.lib import ReadBatch
    cases = _cases(synth_genome)
    batch = ReadBatch.from_list([c[0] for c in cases], quals=[c[1] for c in cases])
    minsc = np.array([_minsc(len(c[0]), local, k) for k, c in enumerate(cases)], dtype=np.int32)
    mask = np.array([(0 if k % 11 == 5 else 1) | (0 if k % 13 == 7 else 2) for k in range(len(cases))], dtype=np.uint8)
    hits, counts = gpu.one_mm(batch, minsc, mask, max_hits=64)
    code = {ord(c): i for i, c in enumerate("ACGTN")}
    nhit = 0
    for k, (r, q) in enumerate(cases):
        want = oracle_one_mm(O, local, r, q, int(minsc[k]), not (mask[k] & 1), not (mask[k] & 2))
        got = []
        for task in range(4):
            for h in hits[k, task, :counts[k, task]]:
                got.append((int(h["top"]), int(h["bot"]), int(h["pos"]), int(h["chr"]), int(h["qchr"]), int(h["score"]), int(task < 2)))
        want = [(t, b, p, code[c], code[qc], s, fw) for (t, b, p, c, qc, s, fw) in want]
        # the reference appends per (strand, index) pass in loop order; the kernel keeps one list per pass
        assert got == want, (k, len(r), got, want)
        nhit += len(got)
    assert nhit > 50
