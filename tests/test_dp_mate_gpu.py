"""GPU parity of the end-to-end DP on mate-finding rectangles (PairedEndPolicy::otherMate + frameFindMateRect): wide windows
in which most rows below the top row block fall under the floor, so the row-block fill skips most of them.  Against the
unmodified reference SwAligner, with the checks of test_dp_gpu._check."""
import numpy as np
import pytest

from bowtie2_b200 import policy, synth
from bowtie2_b200.lib import DP_PROBLEM
from conftest import _build_index
from oracle_lib import Reference, have_reference
from test_dp_gpu import _check

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

UNIT, SPACER, COPIES = 170, 40, 4       # a tandem family: several live bands in one mate window
TANDEM_AT, NGAP_AT, NGAP_LEN = 10000, 20000, 50


def _mutate(rng, seq, n):
    s = seq.copy()
    for p in rng.integers(0, len(s), n):
        s[p] = (s[p] + 1 + rng.integers(0, 3)) % 4
    return s


@pytest.fixture(scope="module")
def mate_genome():
    return make_mate_genome()


def make_mate_genome():
    rng = np.random.default_rng(2026)
    c0 = rng.integers(0, 4, 30000).astype(np.uint8)
    unit = rng.integers(0, 4, UNIT).astype(np.uint8)
    pos = TANDEM_AT
    for k in range(COPIES):
        c0[pos:pos + UNIT] = _mutate(rng, unit, k)          # copy k carries k substitutions: bands of different scores
        pos += UNIT + SPACER
    c0[NGAP_AT:NGAP_AT + NGAP_LEN] = 4
    c1 = rng.integers(0, 4, 3000).astype(np.uint8)          # short: windows off either end
    return [c0, c1]


@pytest.fixture(scope="module")
def mate_index(tmp_path_factory, mate_genome):
    d = tmp_path_factory.mktemp("mate_dp")
    fa = str(d / "g.fa")
    synth.write_fasta(fa, mate_genome)
    base = str(d / "g")
    _build_index("bowtie2-build-s", fa, base)
    return base


def _indel(rng, seq):
    p = int(rng.integers(10, len(seq) - 10))
    k = int(rng.integers(1, 4))
    if rng.integers(0, 2):
        return np.concatenate([seq[:p], rng.integers(0, 4, k).astype(np.uint8), seq[p:]])
    return np.concatenate([seq[:p], seq[p + k:]])


def _mate_problems(genome, L, sc, rng, minsc_bump=0):
    """Anchors of four kinds (true mate inside the window, tandem family, random mate, N gap / reference ends); for each, the
    mate window the reference would search and a mate read of length about L."""
    pe = policy.PairedEndPolicy()
    anchors = []                                                     # (contig, anchor offset, anchor fw, kind)
    c0len, c1len = len(genome[0]), len(genome[1])
    for _ in range(24):
        anchors.append((0, int(rng.integers(300, c0len - 800)), bool(rng.integers(0, 2)), "true"))
    for d in (60, 140, 230):
        anchors.append((0, TANDEM_AT - d - L, True, "tandem"))
        anchors.append((0, TANDEM_AT + COPIES * (UNIT + SPACER) + d, False, "tandem"))
    for _ in range(6):
        anchors.append((0, int(rng.integers(300, c0len - 800)), bool(rng.integers(0, 2)), "random"))
    for d in (-300, -150, 0, 100):
        anchors.append((0, NGAP_AT + d, True, "true"))
    for off in (0, 5, 40):
        anchors.append((1, off, False, "true"))                      # mate window off the left end
        anchors.append((1, c1len - L - off, True, "true"))           # off the right end
    reads, quals, probs, meta = [], [], [], []
    for c, off, fw, kind in anchors:
        tlen = len(genome[c])
        om = pe.other_mate(True, fw, off, -1, tlen, L, L)
        if om is None:
            continue
        oleft, oll, olr, orl, orr, ofw = om
        frag = int(rng.integers(200, 480))
        ms = off + L - frag if oleft else off + frag - L
        if kind == "tandem":
            ms = TANDEM_AT + int(rng.integers(0, COPIES)) * (UNIT + SPACER) + int(rng.integers(-5, 6))
        if kind == "random" or ms < 0 or ms + L > tlen:
            r = rng.integers(0, 4, L).astype(np.uint8)
        else:
            r = genome[c][ms:ms + L].copy()
            r[r > 3] = int(rng.integers(0, 4))
            r = _mutate(rng, r, int(rng.integers(0, 3)))
            if rng.integers(0, 4) == 0:
                r = _indel(rng, r)
            if not ofw:
                r = synth.revcomp(r)
        rdlen = len(r)
        minsc = sc.min_score(rdlen) + minsc_bump
        if minsc > sc.perfect_score(rdlen):
            continue
        found, rect = policy.frame_find_mate_rect(not oleft, oll, olr, orl, orr, rdlen, tlen, sc.max_read_gaps(minsc, rdlen),
                                                  sc.max_ref_gaps(minsc, rdlen), sc.n_ceil(rdlen))
        if not found:
            continue
        probs.append((len(reads), int(ofw), c, rect.refl, rect.refr, rect.triml, rect.corel, rect.corer,
                      minsc, sc.n_ceil_raw(rdlen), 0))
        meta.append((tlen, rect, minsc))
        reads.append(r)
        quals.append(rng.integers(35, 74, rdlen).astype(np.uint8))
    return reads, quals, np.array(probs, dtype=DP_PROBLEM), meta


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("L", [33, 64, 65, 100, 129, 150, 250])
def test_dp_mate_rectangles_match_reference(gpu, mate_index, mate_genome, L):
    gpu.load_index_files(mate_index)
    gpu.set_scoring(local=False)
    R = Reference(mate_index)
    sc = policy.Scoring.default(False)
    rng = np.random.default_rng(L)
    reads, quals, probs, meta = _mate_problems(mate_genome, L, sc, rng)
    assert np.median([m[1].refr - m[1].refl + 1 for m in meta]) > 2 * L   # mate windows, not seed-extension rectangles
    nfound, naln, ngap = _check(gpu, R, mate_genome, reads, quals, probs, meta)
    assert nfound > 20 and naln > 20
    reads, quals, probs, meta = _mate_problems(mate_genome, L, sc, rng, minsc_bump=max(4, L // 10))
    _check(gpu, R, mate_genome, reads, quals, probs, meta)
