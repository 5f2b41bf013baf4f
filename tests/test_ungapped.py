"""SwAligner::ungappedAlign: C restatement vs reference (CPU) and CUDA vs restatement (GPU)."""
import numpy as np
import pytest

from bowtie2_b200 import synth
import oracle_lib
from oracle_lib import Oracle, Reference, have_reference, oracle_ungapped, ref_ungapped, scoring_grid

# the scorings of oracle_lib.scoring_grid() that the ungapped aligner reads: mismatch and N penalties, the N ceiling, the match bonus
GRID = ["mp6,6", "mp2,2", "mp8,3", "np0", "np3", "nceil-L0,0", "nceil-L0,0.5", "local-ma1", "local-ma3"]


def _cases(genome, n=400, seed=77):
    """(read codes, quals, fw, tidx, off, tlen, ohang, minsc-by-mode) around true loci, with substitutions,
    Ns, offsets shifted off the locus, and placements hanging over both reference ends."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        ln = int(rng.choice([20, 33, 50, 100, 150]))
        t = int(rng.integers(0, len(genome)))
        g = genome[t]
        tlen = len(g)
        if k % 9 == 0:
            p = int(rng.choice([-3, -1, 0, tlen - ln, tlen - ln + 2, tlen - ln + 5]))
        else:
            p = int(rng.integers(0, tlen - ln))
        lo, hi = max(p, 0), min(p + ln, tlen)
        r = np.full(ln, 0, dtype=np.uint8)
        r[lo - p:hi - p] = np.minimum(g[lo:hi], 3)
        nsub = int(rng.choice([0, 0, 1, 2, 4, 8]))
        for q in rng.choice(ln, size=nsub, replace=False):
            r[q] = (r[q] + rng.integers(1, 4)) % 4
        if k % 7 == 2:
            r[rng.integers(0, ln)] = 4
        fw = bool(rng.integers(0, 2))
        read = r if fw else synth.revcomp(r)
        qual = rng.integers(33, 74, size=ln).astype(np.uint8)
        off = p + (int(rng.integers(-2, 3)) if k % 11 == 5 else 0)
        out.append((read.astype(np.uint8), qual, fw, t, off, tlen, bool(k % 2)))
    return out


def _minsc(ln, local, k):
    if local:
        return (int(20 + 8.0 * np.log(ln)), ln, 2 * ln - 8)[k % 3]
    return (int(-0.6 - 0.6 * ln), -6, -18)[k % 3]


def _ref_view(rc, d, ln, fw):
    """reference result -> (score, refoff, rowi, rowf, ns, refns, edit rows)"""
    if rc != 1:
        return rc
    rowi = d["trim5"] if fw else d["trim3"]
    rowf = ln - 1 - (d["trim3"] if fw else d["trim5"])
    # Edit::pos starts as the row (aligner_sw.cpp:441), AlnRes::setShape shifts it by the leading trim
    # (aligner_result.cpp:94-110) and invertEdits flips it within the aligned extent for the reverse strand
    rows = sorted((rowi + e[0] if fw else rowf - e[0]) for e in d["edits"])
    return (d["score"], d["refoff"], rowi, rowf, d["ns"], d["refns"], rows)


def _oracle_vs_reference(O, R, local, genome):
    seen = set()
    for k, (r, q, fw, t, off, tlen, ohang) in enumerate(_cases(genome)):
        minsc = _minsc(len(r), local, k)
        rc, d = ref_ungapped(R, local, r, q, fw, t, off, tlen, ohang, minsc)
        oc, od = oracle_ungapped(O, local, r, q, fw, t, off, tlen, ohang, minsc)
        assert oc == rc, (k, oc, rc)
        seen.add(rc)
        if rc == 1:
            want = _ref_view(rc, d, len(r), fw)
            got = (od["score"], off + od["rowi"], od["rowi"], od["rowf"], od["ns"], od["refns"], sorted(np.nonzero(od["mask"])[0].tolist()))
            assert got == want, (k, got, want)
    return seen


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("local", [False, True])
def test_ungapped_oracle_vs_reference(local, synth_index, synth_genome):
    seen = _oracle_vs_reference(Oracle(synth_index), Reference(synth_index), local, synth_genome)
    assert 0 in seen and 1 in seen and (not local or -1 in seen or True)


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", GRID)
def test_ungapped_oracle_vs_reference_under_scoring(name, synth_index, synth_genome):
    sc = scoring_grid()[name]
    O, R = Oracle(synth_index), Reference(synth_index)
    R.set_scoring(sc)
    oracle_lib.SCORING_OVERRIDE = sc
    try:
        seen = _oracle_vs_reference(O, R, sc.local, synth_genome)
    finally:
        oracle_lib.SCORING_OVERRIDE = None
    assert 0 in seen and 1 in seen


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("which,local,scoring", [pytest.param("small", False, None, id="small-False"), pytest.param("small", True, None, id="small-True"),
                                                 pytest.param("large", False, None, id="large-False")] +
                         [pytest.param("small", name.startswith("local"), name, id="small-" + name) for name in ("mp8,3", "mp2,2", "np0", "nceil-L0,0", "local-ma3")])
def test_ungapped_gpu_vs_oracle(which, local, scoring, gpu, synth_index, synth_index_large, synth_genome):
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
    from bowtie2_b200.lib import ReadBatch, UNGAPPED_PROBLEM
    cases = _cases(synth_genome)
    batch = ReadBatch.from_list([c[0] for c in cases], quals=[c[1] for c in cases])
    probs = np.zeros(len(cases), dtype=UNGAPPED_PROBLEM)
    for k, (r, q, fw, t, off, tlen, ohang) in enumerate(cases):
        probs[k] = (k, int(fw), t, off, tlen, _minsc(len(r), local, k), int(ohang))
    res, mask = gpu.ungapped(batch, probs)
    nfound = 0
    for k, (r, q, fw, t, off, tlen, ohang) in enumerate(cases):
        oc, od = oracle_ungapped(O, local, r, q, fw, t, off, tlen, ohang, int(probs[k]["minsc"]))
        g = res[k]
        assert int(g["status"]) == oc, (k, g, oc)
        if oc == 1:
            nfound += 1
            assert (int(g["score"]), int(g["rowi"]), int(g["rowf"]), int(g["ns"]), int(g["refns"]), int(g["nedits"])) == \
                   (od["score"], od["rowi"], od["rowf"], od["ns"], od["refns"], od["nedits"]), k
            assert np.array_equal(mask[k, :len(r)], od["mask"]), k
    assert nfound > 50
