"""GPU parity for K3: the CUDA DP (fill + gather + backtrace) through the C ABI vs the unmodified
reference SwAligner (oracle/_ref glue): found/best, the full candidate list, every alignment's
score / offset / gaps / Ns and its edit list."""
import numpy as np
import pytest

from bowtie2_b200 import policy, synth
from bowtie2_b200.lib import DP_PROBLEM, ReadBatch, ops_to_edits
import oracle_lib
from oracle_lib import Oracle, Reference, have_reference, oracle_dp, ref_dp, scoring_grid

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def _problems(genome, reads, truth, sc, jitter_rng, minsc_bump=0):
    """One seed-extension DP per alignable read, framed as SwDriver::extendSeeds would
    (aligner_sw_driver.cpp:1185-1283), with the seed diagonal jittered by a few bases."""
    probs, meta = [], []
    for i, (r, (c, p, strand)) in enumerate(zip(reads, truth)):
        if c < 0:
            c, p, strand = 0, int(jitter_rng.integers(0, len(genome[0]) - len(r))), 1
        rdlen = len(r)
        minsc = sc.min_score(rdlen) + minsc_bump
        if minsc > sc.perfect_score(rdlen):
            continue
        off = p + int(jitter_rng.integers(-3, 4))
        tlen = len(genome[c])
        found, rect = policy.frame_seed_extension_rect(off, rdlen, tlen, sc.max_read_gaps(minsc, rdlen),
                                                       sc.max_ref_gaps(minsc, rdlen), sc.n_ceil(rdlen))
        if not found:
            continue
        probs.append((i, 1 if strand > 0 else 0, c, rect.refl, rect.refr, rect.triml, rect.corel, rect.corer,
                      minsc, sc.n_ceil_raw(rdlen), 0))
        meta.append((tlen, rect, minsc))
    return np.array(probs, dtype=DP_PROBLEM), meta


def _check(gpu, R, genome, reads, quals, probs, meta, local=False, max_cands=None, sc=None, wants=None):
    """bt2g_dp_extend against ref_dp problem by problem.  sc: a policy.Scoring the caller installed on both sides
    (gpu.set_scoring_policy, R.set_scoring), which also sizes the op rows; wants: a dict that keeps the reference's answers
    across calls on the same problems"""
    batch = ReadBatch.from_list(reads, quals)
    max_ops = int(batch.lengths().max()) + 80
    if sc is not None:
        local = sc.local
        max_ops = max([max_ops] + [len(reads[int(p["read_idx"])]) + sc.max_read_gaps(int(p["minsc"]), len(reads[int(p["read_idx"])])) for p in probs])
    summ, cands, alns, ops = gpu.dp_extend(batch, probs, max_cands=max_cands or (8192 if local else 256),
                                           max_alns=32 if sc is not None else (24 if local else 8), max_ops=max_ops)
    nfound = naln = ngap = 0
    for k, pr in enumerate(probs):
        tlen, rect, minsc = meta[k]
        i = int(pr["read_idx"])
        want = None if wants is None else wants.get(k)
        if want is None:
            want = ref_dp(R, local, reads[i], quals[i], int(pr["fw"]), int(pr["tidx"]), tlen, rect, minsc, max_cands=max(16384, max_cands or 0),
                          max_alns=64, max_edits=16384)
            if wants is not None:
                wants[k] = want
        s = summ[k]
        assert s["flags"] == 0, (k, s)
        assert bool(s["found"]) == bool(want["found"]), (k, s, want["found"], want["best"])
        if not want["found"]:
            # below minsc the reference's number is a saturated 8/16-bit value (0xff-biased u8 clamps
            # at -255, aligner_swsse_ee_u8.cpp:1119-1131); only "not found" is comparable
            assert s["best"] < minsc
            continue
        nfound += 1
        assert s["best"] == want["best"]
        assert s["ncand"] == want["ncand"]
        got_c = [(int(c["row"]), int(c["col"]), int(c["score"])) for c in cands[k][:s["ncand"]]]
        assert got_c == want["cands"], (k, got_c[:5], want["cands"][:5])
        assert s["naln"] == want["naln"], (k, s["naln"], want["naln"])
        for a_i, wa in enumerate(want["alns"]):
            a = alns[k][a_i]
            assert (int(a["score"]), int(a["ns"]), int(a["gaps"])) == (wa["score"], wa["ns"], wa["gaps"]), (k, a, wa)
            assert int(pr["refl"]) + int(a["col0"]) == wa["refoff"], (k, a, wa)
            ed = ops_to_edits(ops[k][a_i], int(a["nops"]), reads[i], bool(pr["fw"]), int(a["row0"]), int(a["trim_end"]))
            t5, t3 = (int(a["trim_beg"]), int(a["trim_end"])) if pr["fw"] else (int(a["trim_end"]), int(a["trim_beg"]))
            assert (t5, t3) == (wa["trim5"], wa["trim3"]), (k, a, wa)
            assert ed == wa["edits"], (k, a_i, ed, wa["edits"])
            naln += 1
            ngap += wa["gaps"] > 0
    return nfound, naln, ngap


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("rdlen,sub,indel", [(100, 0.01, 0.002), (150, 0.02, 0.004), (50, 0.01, 0.0), (250, 0.01, 0.003), (33, 0.03, 0.01),
                                             (128, 0.01, 0.003), (129, 0.02, 0.003), (180, 0.01, 0.004), (200, 0.015, 0.003)])
def test_dp_e2e_matches_reference(gpu, synth_index, synth_genome, rdlen, sub, indel):
    gpu.load_index_files(synth_index)
    gpu.set_scoring(local=False)
    R = Reference(synth_index)
    sc = policy.Scoring.default(False)
    reads, quals, truth = synth.make_reads(synth_genome, 250, rdlen, seed=rdlen, sub_rate=sub, indel_rate=indel, random_frac=0.05)
    rng = np.random.default_rng(rdlen)
    for r in reads[:25]:
        r[rng.integers(0, len(r))] = 4                       # Ns in reads
    probs, meta = _problems(synth_genome, reads, truth, sc, rng)
    nfound, naln, ngap = _check(gpu, R, synth_genome, reads, quals, probs, meta)
    assert nfound > 100 and naln > 100
    if indel > 0:
        assert ngap > 0


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("mode", ["0", "1"])
def test_dp_e2e_kernel_generations(gpu, synth_index, synth_genome, mode):
    """The move-code end-to-end DP kernels stay correct: mode 1 (s16x2) runs when a batch's score range does not fit the bytes
    of the split H-byte kernels, mode 0 (32-bit) when it does not fit s16x2 either or under a mode cap of 0.  The context's mode
    cap (bt2g_set_dp_mode) selects them here: a 100 bp read's default minimum score fits a byte, so each cap is the mode that
    runs."""
    gpu.load_index_files(synth_index)
    gpu.set_scoring(local=False)
    R = Reference(synth_index)
    sc = policy.Scoring.default(False)
    reads, quals, truth = synth.make_reads(synth_genome, 120, 100, seed=900 + int(mode), sub_rate=0.02, indel_rate=0.004)
    probs, meta = _problems(synth_genome, reads, truth, sc, np.random.default_rng(5))
    assert _kernel_mode(sc, int(probs["minsc"].min()), 100, int(mode)) == int(mode)
    gpu.set_dp_mode(int(mode))
    try:
        nfound, naln, ngap = _check(gpu, R, synth_genome, reads, quals, probs, meta)
    finally:
        gpu.set_dp_mode(3)
    assert nfound > 80 and ngap > 3


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
def test_dp_e2e_edges(gpu, synth_index, synth_genome):
    """Windows hanging off either reference end, spanning the N gap, repeats (many candidates),
    and a tightened minimum score."""
    gpu.load_index_files(synth_index)
    gpu.set_scoring(local=False)
    R = Reference(synth_index)
    sc = policy.Scoring.default(False)
    g = synth_genome
    rng = np.random.default_rng(3)
    reads, quals, truth = [], [], []
    L = 100
    glen = len(g[0])
    for p in [0, 1, 5, 29, 31, glen - L, glen - L - 1, glen - L - 31, glen // 2 - 60, glen // 2 - 20, glen // 2 + 10]:
        for strand in (1, -1):
            r = g[1][p:p + L].copy()
            r[r > 3] = 0
            r[rng.integers(0, L)] ^= 1
            reads.append(r if strand > 0 else synth.revcomp(r))
            quals.append(rng.integers(35, 74, L).astype(np.uint8))
            truth.append((1, p, strand))
    probs, meta = _problems(g, reads, truth, sc, rng)
    _check(gpu, R, g, reads, quals, probs, meta)
    probs, meta = _problems(g, reads, truth, sc, rng, minsc_bump=40)
    _check(gpu, R, g, reads, quals, probs, meta)


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("rdlen,sub,indel", [(100, 0.02, 0.003), (150, 0.03, 0.005), (300, 0.02, 0.004), (60, 0.02, 0.0)])
def test_dp_local_matches_reference(gpu, synth_index, synth_genome, rdlen, sub, indel):
    """--local: floors at 0, candidates anywhere in the rectangle, soft trimming, domination filter."""
    gpu.load_index_files(synth_index)
    gpu.set_scoring(local=True)
    R = Reference(synth_index)
    sc = policy.Scoring.default(True)
    reads, quals, truth = synth.make_reads(synth_genome, 160, rdlen, seed=7 * rdlen, sub_rate=sub, indel_rate=indel, random_frac=0.05)
    rng = np.random.default_rng(rdlen + 1)
    for i, r in enumerate(reads):
        if i % 3 == 0:                                   # junk ends -> soft clipping
            k = int(rng.integers(3, max(4, rdlen // 5)))
            r[:k] = rng.integers(0, 4, k)
        if i % 4 == 0:
            k = int(rng.integers(3, max(4, rdlen // 5)))
            r[-k:] = rng.integers(0, 4, k)
        if i % 11 == 0:
            r[rng.integers(0, rdlen)] = 4
    probs, meta = _problems(synth_genome, reads, truth, sc, rng)
    nfound, naln, ngap = _check(gpu, R, synth_genome, reads, quals, probs, meta, local=True)
    assert nfound > 100 and naln > 100
    gpu.set_scoring(local=False)


def _kernel_mode(sc, min_minsc, max_len, cap):
    """dp_kernel_mode (dp_device.cuh): the end-to-end generation bt2g_dp_extend runs under the mode cap; "local" for local scoring"""
    if sc.local:
        return "local"
    if cap == 0 or min_minsc < -8000 or sc.match_bonus * max_len > 8000:
        return 0
    rng = sc.match_bonus * max_len - (min_minsc - sc.match_bonus - 1)
    return 3 if cap >= 3 and rng <= 127 else 1


def _rows_per_lane(max_len, mode):
    """dp_rows_per_lane (dp_device.cuh); the local kernels use the move-code rows"""
    if mode == 3:
        return next(r for r in (4, 5, 6, 8, 10, 12, 16) if 32 * r >= max_len)
    return 4 if max_len <= 128 else (8 if max_len <= 256 else 16)


GRID_LENGTHS = [100, 150, 180, 250]        # 32 R >= length: R = 4, 5, 6, 8 on the H-byte kernels, 4 and 8 on the move-code kernels
GRID_RAN = set()                           # (mode, rows per lane) of the grid's calls with found alignments


@pytest.fixture(scope="module")
def grid_mate_index(tmp_path_factory):
    """the mate-window genome of test_dp_mate_gpu (tandem family, N gap, a short contig) and its index"""
    import test_dp_mate_gpu
    from conftest import _build_index
    genome = test_dp_mate_gpu.make_mate_genome()
    d = tmp_path_factory.mktemp("grid_mate")
    synth.write_fasta(str(d / "g.fa"), genome)
    _build_index("bowtie2-build-s", str(d / "g.fa"), str(d / "g"))
    return genome, str(d / "g")


def _grid_reads(genome, sc, L, seed, n_rich):
    reads, quals, truth = synth.make_reads(genome, 40, L, seed=seed, sub_rate=0.02, indel_rate=0.006, random_frac=0.05)
    rng = np.random.default_rng(seed)
    for r in reads[:6]:
        r[rng.integers(0, L)] = 4
    if n_rich:
        for r in reads[::2]:
            r[rng.integers(0, L, int(rng.integers(1, 6)))] = 4
    if sc.local:
        for r in reads[::3]:
            k = int(rng.integers(3, 15))
            r[:k] = rng.integers(0, 4, k)
    return reads, quals, truth, rng


def _byte_bump(sc, L):
    """end-to-end minimum scores below -127 are raised to -100 at the longest grid length, so that its rows-per-lane instantiation
    of the H-byte kernels runs too (the move-code kernels run at every length)"""
    return 0 if sc.local or sc.min_score(L) >= -127 or L < 250 else -100 - sc.min_score(L)


def _caps_checked(gpu, R, genome, reads, quals, probs, meta, sc, L):
    """the problems at every mode cap (local: its one generation), each against the reference; -> found problems per cap"""
    found, wants = [], {}
    for cap in ((3,) if sc.local else (0, 1, 3)):
        gpu.set_dp_mode(cap)
        nfound, naln, _ = _check(gpu, R, genome, reads, quals, probs, meta, sc=sc, max_cands=16384 if sc.local else 2048, wants=wants)
        mode = _kernel_mode(sc, int(probs["minsc"].min()), max(len(reads[int(i)]) for i in probs["read_idx"]), cap)
        if nfound:
            GRID_RAN.add((mode, _rows_per_lane(max(len(reads[int(i)]) for i in probs["read_idx"]), 0 if mode == "local" else mode)))
        found.append((cap, mode, nfound, naln))
    return found


def _fates(gpu, O, reads, quals, probs, meta, sc, cap):
    """candidate fates (SUCCEEDED / FAILED exactly where the reference starts a backtrace, in order) against oracle_dp's attempt log"""
    gpu.set_dp_mode(cap)
    summ, cands, _, _ = gpu.dp_extend(ReadBatch.from_list(reads, quals), probs, max_cands=32768 if sc.local else 2048, max_alns=32,
                                      max_ops=max(len(r) for r in reads) + sc.max_read_gaps(int(probs["minsc"].min()), max(len(r) for r in reads)))
    n_att = 0
    for k, p in enumerate(probs):
        i = int(p["read_idx"])
        assert summ[k]["flags"] == 0, (k, summ[k])
        d = oracle_dp(O, sc.local, reads[i], quals[i], bool(p["fw"]), int(p["tidx"]), meta[k][1], int(p["minsc"]), int(p["nceil"]),
                      max_cands=65536, max_alns=64, max_edits=16384, attempts=True)
        assert bool(summ[k]["found"]) == bool(d["found"]), k
        if not d["found"]:
            continue
        got = [(ci, int(cands[k][ci]["fate"])) for ci in range(int(summ[k]["ncand"])) if int(cands[k][ci]["fate"]) in (2, 3)]
        want = [(ci, 3 if ai >= 0 else 2) for (_, ai), ci in zip(d["attempts"], d["attempt_cands"])]
        assert got == want, (k, got[:6], want[:6])
        n_att += len(want)
    return n_att


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", sorted(scoring_grid()))
def test_dp_matches_reference_under_scoring(gpu, synth_index, synth_genome, grid_mate_index, name):
    """Every DP kernel generation (mode caps 0, 1 and 3) at R = 4, 5, 6 and 8 on seed-extension rectangles, and on mate windows at 150 bp,
    against SwAligner under oracle_lib.scoring_grid()'s scorings; candidate fates against the C restatement's attempt log in
    modes 1 and 3 (local: its kernel)"""
    from test_dp_mate_gpu import _mate_problems
    sc = scoring_grid()[name]
    mate_genome, mate_base = grid_mate_index
    default = policy.Scoring.default(sc.local)
    try:
        gpu.load_index_files(synth_index)
        gpu.set_scoring_policy(sc)
        R = Reference(synth_index)
        R.set_scoring(sc)
        seeds = 0
        for L in GRID_LENGTHS:
            reads, quals, truth, rng = _grid_reads(synth_genome, sc, L, 300 + L, name.startswith("nceil"))
            probs, meta = _problems(synth_genome, reads, truth, sc, rng, minsc_bump=_byte_bump(sc, L))
            per_cap = _caps_checked(gpu, R, synth_genome, reads, quals, probs, meta, sc, L)
            assert all(nf > 10 and na > 10 for _, _, nf, na in per_cap), (L, per_cap)
            seeds += per_cap[0][2]
            if L == 100:
                O = Oracle(synth_index)
                oracle_lib.SCORING_OVERRIDE = sc
                for cap in ((3,) if sc.local else (1, 3)):
                    assert _fates(gpu, O, reads, quals, probs, meta, sc, cap) > 20
                oracle_lib.SCORING_OVERRIDE = None
        if name == "minsc-126":
            assert per_cap[-1][1] == 3                              # 1 - minsc = 127: the H-byte kernels
        if name == "minsc-127":
            assert per_cap[-1][1] == 1                              # 128: the s16x2 move-code kernel
        R.set_scoring(default)
        gpu.load_index_files(mate_base)
        gpu.set_scoring_policy(sc)
        R = Reference(mate_base)
        R.set_scoring(sc)
        reads, quals, probs, meta = _mate_problems(mate_genome, 150, sc, np.random.default_rng(150))
        per_cap = _caps_checked(gpu, R, mate_genome, reads, quals, probs, meta, sc, 150)
        assert all(nf > 5 and na > 5 for _, _, nf, na in per_cap), per_cap
        R.set_scoring(default)
    finally:
        oracle_lib.SCORING_OVERRIDE = None
        gpu.set_dp_mode(3)
        gpu.set_scoring(local=False)


def test_dp_zz_every_grid_generation_ran():
    """the end of the file: under the scoring grid every end-to-end generation ran with found alignments at every rows-per-lane
    instantiation that reads of 100-250 bases reach, and the local kernel at both of its"""
    want = {(0, 4), (0, 8), (1, 4), (1, 8)} | {(3, r) for r in (4, 5, 6, 8)} | {("local", 4), ("local", 8)}
    assert want <= GRID_RAN, sorted(want - GRID_RAN, key=str)
