"""GPU parity of the split end-to-end DP (fill + tail, bt2g_dp_extend) at the edges of its geometry: read lengths around the row
counts that a row block, a lane and a warp's rows divide (multiples of 16, 32, 48 and 64), chunks whose problem count leaves a
packed slot or a warp's second pair idle, problems of very different widths side by side, a bad-shape problem among good ones,
and a match bonus (full-width blocks).  Against the unmodified reference SwAligner with the checks of test_dp_gpu._check, or,
with a match bonus, against the recorded results of the fused H-byte kernel."""
import os

import numpy as np
import pytest

from bowtie2_b200 import policy, synth
from bowtie2_b200.lib import ReadBatch
from conftest import GOLDEN
from oracle_lib import Reference, have_reference
from test_dp_gpu import _check, _problems
from test_dp_mate_gpu import _mate_problems, mate_genome, mate_index  # noqa: F401  (fixtures)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

EDGE_LENGTHS = [15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65, 95, 96, 97, 127, 128, 129, 143, 144, 145, 150, 200, 250]


def _short_mates(monkeypatch, L):
    """test_dp_mate_gpu's indels need 21 bases or more: shorter mates keep substitutions only"""
    if L < 24:
        import test_dp_mate_gpu
        monkeypatch.setattr(test_dp_mate_gpu, "_indel", lambda rng, seq: seq)


def _seed_problems(genome, L, sc, rng, n):
    reads, quals, truth = synth.make_reads(genome, n, L, seed=1000 + L, sub_rate=0.02, indel_rate=0.004 if L > 20 else 0.0,
                                           random_frac=0.05)
    probs, meta = _problems(genome, reads, truth, sc, rng)
    return reads, quals, probs, meta


def _merge(a, b):
    """Two problem sets over one read batch: the reads of b follow those of a."""
    ra, qa, pa, ma = a
    rb, qb, pb, mb = b
    pb = pb.copy()
    pb["read_idx"] += len(ra)
    return ra + rb, qa + qb, np.concatenate([pa, pb]), ma + mb


def _interleave(probs, meta, order):
    return probs[order], [meta[i] for i in order]


def _assert_same(a, b):
    """Two dp_extend results agree on everything they report: summaries, candidates, alignments and op strings."""
    (s1, c1, a1, o1), (s2, c2, a2, o2) = a, b
    assert len(s1) == len(s2)
    for f in ("found", "best", "ncand", "naln", "flags"):
        assert np.array_equal(s1[f], s2[f]), f
    for k in range(len(s1)):
        nc, na = int(s1["ncand"][k]), int(s1["naln"][k])
        assert c1[k][:nc].tobytes() == c2[k][:nc].tobytes(), k
        assert a1[k][:na].tobytes() == a2[k][:na].tobytes(), k
        for i in range(na):
            n = int(a1[k][i]["nops"])
            assert o1[k][i][:n].tobytes() == o2[k][i][:n].tobytes(), (k, i)


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("L", EDGE_LENGTHS)
def test_dp_block_edges_match_reference(gpu, mate_index, mate_genome, L, monkeypatch):
    """Seed-extension and mate-finding rectangles at read lengths around the block edges, mixed so that each warp carries narrow
    and wide windows; the batch is cut to problem counts of 1, 2 and 3 mod 4."""
    _short_mates(monkeypatch, L)
    gpu.load_index_files(mate_index)
    gpu.set_scoring(local=False)
    R = Reference(mate_index)
    sc = policy.Scoring.default(False)
    rng = np.random.default_rng(4800 + L)
    reads, quals, probs, meta = _merge(_seed_problems(mate_genome, L, sc, rng, 40), _mate_problems(mate_genome, L, sc, rng))
    assert len(probs) > 24
    # narrow and wide windows alternate: every warp holds windows of very different widths
    widths = probs["refr"] - probs["refl"]
    by_w = list(np.argsort(widths, kind="stable"))
    order = [by_w.pop(0) if k % 2 == 0 else by_w.pop() for k in range(len(by_w))]
    probs, meta = _interleave(probs, meta, order)
    nfound = naln = 0
    for cut in (len(probs) - (len(probs) - 1) % 4, 6, 3):      # counts = 1, 2, 3 (mod 4)
        f, a, _ = _check(gpu, R, mate_genome, reads, quals, probs[:cut], meta[:cut])
        nfound += f; naln += a
    assert nfound > 10 and naln > 10


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("L", [48, 150])
def test_dp_bad_shape_among_good(gpu, mate_index, mate_genome, L):
    """One problem with an empty window in every group of four: it is flagged, and the problems packed and swept beside it still
    match the reference."""
    gpu.load_index_files(mate_index)
    gpu.set_scoring(local=False)
    R = Reference(mate_index)
    sc = policy.Scoring.default(False)
    rng = np.random.default_rng(77 + L)
    reads, quals, probs, meta = _mate_problems(mate_genome, L, sc, rng)
    probs = probs[:len(probs) // 4 * 4].copy()
    meta = meta[:len(probs)]
    bad = np.arange(len(probs)) % 4 == (np.arange(len(probs)) // 4) % 4        # a different slot of each quad
    probs["refr"][bad] = probs["refl"][bad] - 1
    batch = ReadBatch.from_list(reads, quals)
    summ, _, _, _ = gpu.dp_extend(batch, probs, max_cands=256, max_alns=8, max_ops=L + 80)
    assert np.all(summ["flags"][bad] == 1) and not np.any(summ["found"][bad])
    good = np.nonzero(~bad)[0]
    _check(gpu, R, mate_genome, reads, quals, probs[good], [meta[i] for i in good])
    # the same problems with the bad ones in place give the same results as without them
    full = gpu.dp_extend(batch, probs, max_cands=256, max_alns=8, max_ops=L + 80)
    _assert_same(tuple(x[good] for x in full), gpu.dp_extend(batch, probs[good], max_cands=256, max_alns=8, max_ops=L + 80))


MATCH_BONUS_LENGTHS = [15, 16, 17, 33, 47, 48, 49, 64]
MATCH_BONUS_GOLDEN = os.path.join(GOLDEN, "dp_match_bonus_hbyte.npz")


def _match_bonus_problems(mate_genome, L, monkeypatch):
    """seed-extension and mate rectangles of reads of L bases under match bonus 1, cut to 3 (mod 4) problems"""
    _short_mates(monkeypatch, L)
    sc = policy.Scoring.default(False)
    sc.match_bonus = 1
    rng = np.random.default_rng(31 + L)
    reads, quals, probs, meta = _merge(_seed_problems(mate_genome, L, sc, rng, 40), _mate_problems(mate_genome, L, sc, rng))
    return ReadBatch.from_list(reads, quals), probs[:len(probs) - (len(probs) - 3) % 4]


def _compact(out):
    """everything a dp_extend result reports (the fields _assert_same compares) as four flat arrays"""
    s, c, a, o = out
    summ = np.stack([s[f].astype(np.int64) for f in ("found", "best", "ncand", "naln", "flags")], axis=1)
    cands = [c[k][:int(s["ncand"][k])] for k in range(len(s))]
    alns = [a[k][:int(s["naln"][k])] for k in range(len(s))]
    ops = [o[k][i][:int(alns[k][i]["nops"])] for k in range(len(s)) for i in range(len(alns[k]))]
    return {"summ": summ, "cands": np.concatenate(cands), "alns": np.concatenate(alns), "ops": np.concatenate(ops)}


@pytest.mark.parametrize("L", MATCH_BONUS_LENGTHS)
def test_dp_match_bonus_same_as_recorded_fused_kernel(gpu, mate_index, mate_genome, L, monkeypatch):
    """With a match bonus every row block sweeps the full width; the split H-byte kernels give what the fused H-byte kernel gave
    on the same problems (the byte encoding holds these short reads' score range).  tests/golden/dp_match_bonus_hbyte.npz holds
    the fused kernel's results, recorded before it was retired.  The move-code kernels are no substitute: they report the exact
    best score of a problem without candidates where the H-byte kernels report the floor, and end-to-end scoring with a match
    bonus, which the reference does not define, lets their backtraces find other alignments."""
    gpu.load_index_files(mate_index)
    gpu.set_scoring(local=False, match_bonus=1)
    batch, probs = _match_bonus_problems(mate_genome, L, monkeypatch)
    try:
        gpu.set_dp_mode(3)
        out = gpu.dp_extend(batch, probs, max_cands=256, max_alns=8, max_ops=L + 80)
    finally:
        gpu.set_scoring(local=False)
    assert int(out[0]["found"].sum()) > 10
    got, want = _compact(out), np.load(MATCH_BONUS_GOLDEN)
    for key, v in got.items():
        w = want[f"{key}_{L}"]
        assert v.dtype == w.dtype and v.shape == w.shape and v.tobytes() == w.tobytes(), key
