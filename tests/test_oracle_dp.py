"""CPU: the plain-C DP restatement (with the reference's full mask / branch-stack backtrace) vs the
unmodified reference SwAligner."""
import numpy as np
import pytest

from bowtie2_b200 import policy, synth
import oracle_lib
from oracle_lib import Oracle, Reference, have_reference, oracle_dp, ref_dp, scoring_grid


def _compare(O, R, genome, sc, rdlen, sub, indel, seed, n_reads=120, n_rich=False):
    """ref_dp against oracle_dp over seed-extension rectangles of reads around their true loci (default and tightened minimum
    scores); oracle_dp runs under SCORING_OVERRIDE = sc, the reference under R.set_scoring(sc).  -> problems with alignments"""
    local = sc.local
    reads, quals, truth = synth.make_reads(genome, n_reads, rdlen, seed=seed, sub_rate=sub, indel_rate=indel, random_frac=0.05)
    rng = np.random.default_rng(rdlen)
    for r in reads[:15]:
        r[rng.integers(0, len(r))] = 4
    if n_rich:
        for r in reads[::2]:
            r[rng.integers(0, len(r), int(rng.integers(1, 6)))] = 4
    if local:
        for r in reads[::3]:
            k = int(rng.integers(3, 12))
            r[:k] = rng.integers(0, 4, k)
    n = nfound = 0
    for i, (r, q, (c, p, strand)) in enumerate(zip(reads, quals, truth)):
        if c < 0:
            c, p, strand = 0, int(rng.integers(0, 30000)), 1
        for bump in (0, 25):
            minsc = sc.min_score(rdlen) + bump
            off = p + int(rng.integers(-3, 4))
            tlen = len(genome[c])
            found, rect = policy.frame_seed_extension_rect(off, rdlen, tlen, sc.max_read_gaps(minsc, rdlen),
                                                           sc.max_ref_gaps(minsc, rdlen), sc.n_ceil(rdlen))
            if not found:
                continue
            if minsc > sc.perfect_score(rdlen):
                continue
            want = ref_dp(R, local, r, q, strand > 0, c, tlen, rect, minsc, max_cands=8192, max_edits=16384)
            got = oracle_dp(O, local, r, q, strand > 0, c, rect, minsc, sc.n_ceil_raw(rdlen), max_cands=8192, max_edits=16384)
            n += 1
            assert got["found"] == want["found"], (i, got, want["found"])
            if not want["found"]:
                assert got["best"] < minsc
                continue
            nfound += 1
            assert got["best"] == want["best"] and got["ncand"] == want["ncand"] and got["cands"] == want["cands"]
            assert got["naln"] == want["naln"]
            for a, b in zip(got["alns"], want["alns"]):
                assert a == b, (i, a, b)
    return nfound


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("local", [False, True])
@pytest.mark.parametrize("rdlen,sub,indel", [(100, 0.015, 0.003), (60, 0.03, 0.01), (180, 0.01, 0.004)])
def test_oracle_dp_matches_reference(synth_index, synth_genome, rdlen, sub, indel, local):
    O, R = Oracle(synth_index), Reference(synth_index)
    assert _compare(O, R, synth_genome, policy.Scoring.default(local), rdlen, sub, indel, 3 * rdlen) > 100


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", sorted(scoring_grid()))
def test_oracle_dp_matches_reference_under_scoring(synth_index, synth_genome, name):
    """the restatement and SwAligner under the same non-default scoring, at 100 bp with substitutions and indels"""
    sc = scoring_grid()[name]
    O, R = Oracle(synth_index), Reference(synth_index)
    R.set_scoring(sc)
    oracle_lib.SCORING_OVERRIDE = sc
    try:
        nfound = _compare(O, R, synth_genome, sc, 100, 0.02, 0.006, 11, n_reads=80, n_rich=name.startswith("nceil"))
    finally:
        oracle_lib.SCORING_OVERRIDE = None
    assert nfound > 40
