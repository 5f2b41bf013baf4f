"""GPU parity of every DP kernel instantiation that reads of 251 to 512 bases reach, and of mate windows up to 8000 columns, against
the unmodified reference SwAligner, with the checks of test_dp_gpu._check (found, best, the full candidate list, alignments, edit
lists, trims).

The reference glue runs default penalties, so the kernel generation of a bt2g_dp_extend call is steered by the problems' minimum
scores and the context's mode cap: under default end-to-end scoring (no match bonus) the default minimum score of a read longer than
about 210 bases puts the whole call on the s16x2 move-code kernel (mode 1); a minimum score of -126 or more fits the score range in a
byte, so the split H-byte fill + tail kernels run (mode 3) unless the cap is below 3.  Reads of 424 bases and more have a
default minimum score below -254, where the reference leaves its u8 matrix for the i16 one; local reads longer than about 127 bases
saturate the reference's u8 local matrix and make it rerun in i16."""
import numpy as np
import pytest

from bowtie2_b200 import policy, synth
from bowtie2_b200.lib import DP_PROBLEM, ReadBatch
from oracle_lib import Reference, have_reference
from test_dp_gpu import _check, _problems
from test_dp_mate_gpu import NGAP_AT, TANDEM_AT, _mate_problems, _mutate, mate_genome, mate_index  # noqa: F401  (fixtures)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800),
              pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")]

LENGTHS = [251, 256, 257, 288, 289, 320, 321, 384, 385, 423, 424, 480, 511, 512]
BYTE_MINSC = -100           # 1 - minsc <= 127: the score range of an end-to-end problem fits the H-byte kernels
SMEM_OPTIN = 227 * 1024     # dynamic shared memory one block may opt in to on sm_90
RAN = set()                 # (mode, rows per lane) of the end-to-end calls with found alignments; ("local", R) for local


def _mode(min_minsc, cap):
    """dp_kernel_mode (dp_device.cuh) under default end-to-end scoring: no match bonus, so the range is 1 - minsc"""
    if cap == 0 or min_minsc < -8000:
        return 0
    return 3 if cap >= 3 and 1 - min_minsc <= 127 else 1


def _rows(max_len, mode):
    """dp_rows_per_lane (dp_device.cuh)"""
    if mode == 3:
        return next(r for r in (4, 5, 6, 8, 10, 12, 16) if 32 * r >= max_len)
    return 4 if max_len <= 128 else (8 if max_len <= 256 else 16)


def _smem_per_warp(max_col):
    """dp_smem_per_warp (dp_kernels.cu)"""
    return (7 * max_col + 31) & ~15


def _fits_four_warps(width, mode, rows):
    """whether the kernels of `mode` fit the block shapes they had before wide windows were sized (4 warps, 8 for the tail) in
    SMEM_OPTIN; max_col = width + 1, as bt2g_dp_extend counts it"""
    m = width + 1
    if mode == 1:
        return 4 * 2 * _smem_per_warp(m) <= SMEM_OPTIN
    if mode == 3:
        prof = (3 * 32 * rows + 15) & ~15
        return 8 * (_smem_per_warp(m) + prof + 16 * 8) <= SMEM_OPTIN
    return 4 * _smem_per_warp(m) <= SMEM_OPTIN


def _fit_512(reads, quals, probs, meta):
    """drops the problems of reads an insertion made longer than 512 bases (bt2g_dp_extend refuses a call that holds one) and cuts
    those reads and their qualities, which no problem uses any more"""
    keep = [k for k, p in enumerate(probs) if len(reads[int(p["read_idx"])]) <= 512]
    for i in range(len(reads)):
        reads[i], quals[i] = reads[i][:512], quals[i][:512]
    return probs[keep], [meta[k] for k in keep]


def _run(gpu, R, genome, reads, quals, probs, meta, cap, local=False):
    """one bt2g_dp_extend call at mode cap `cap`, checked against the reference; returns the (mode, R) it ran and _check's counts"""
    if len(probs) == 0:
        return None, (0, 0, 0)
    gpu.set_dp_mode(cap)
    max_len = max(len(reads[int(i)]) for i in probs["read_idx"])
    if local:
        key = ("local", _rows(max_len, 0))
    else:
        mode = _mode(int(probs["minsc"].min()), cap)
        key = (mode, _rows(max_len, mode))
    try:
        got = _check(gpu, R, genome, reads, quals, probs, meta, local=local, max_cands=65536 if local else 2048)
    finally:
        gpu.set_dp_mode(3)
    if got[0]:
        RAN.add(key)
    return key, got


def _four_calls(gpu, R, genome, make):
    """per length: default minimum score uncapped (mode 1) and capped at 0 (mode 0); a byte-range minimum score uncapped (mode 3)
    and capped at 1 (mode 1).  make(bump) -> (reads, quals, probs, meta) with minsc = default + bump"""
    sc = policy.Scoring.default(False)
    keys, found = [], 0
    for byte_range, cap in [(False, 3), (False, 0), (True, 3), (True, 1)]:
        reads, quals, probs, meta = make(sc, byte_range)
        key, (nfound, naln, _) = _run(gpu, R, genome, reads, quals, probs, meta, cap)
        keys.append(key)
        found += nfound
        assert nfound > 5 and naln > 5, (key, nfound, naln)
    return keys, found


@pytest.mark.parametrize("L", LENGTHS)
def test_long_seed_rectangles_match_reference(gpu, synth_index, synth_genome, L):
    gpu.load_index_files(synth_index)
    gpu.set_scoring(local=False)
    R = Reference(synth_index)

    def make(sc, byte_range):
        reads, quals, truth = synth.make_reads(synth_genome, 40, L, seed=L, sub_rate=0.01, indel_rate=0.003, random_frac=0.05)
        rng = np.random.default_rng(L)
        for r in reads[:8]:
            r[rng.integers(0, L, 2)] = 4                                  # Ns in reads
        bump = BYTE_MINSC - sc.min_score(L) if byte_range else 0
        probs, meta = _problems(synth_genome, reads, truth, sc, rng, minsc_bump=bump)
        return reads, quals, probs, meta
    keys, _ = _four_calls(gpu, R, synth_genome, make)
    assert keys == [(1, _rows(L, 1)), (0, _rows(L, 0)), (3, _rows(L, 3)), (1, _rows(L, 1))], keys


@pytest.mark.parametrize("L", LENGTHS)
def test_long_mate_rectangles_match_reference(gpu, mate_index, mate_genome, L):
    """mate windows (reference ends, the N gap, a tandem family) of reads of about L bases"""
    gpu.load_index_files(mate_index)
    gpu.set_scoring(local=False)
    R = Reference(mate_index)

    def make(sc, byte_range):
        rng = np.random.default_rng(L)
        reads, quals, probs, meta = _mate_problems(mate_genome, L, sc, rng, minsc_bump=BYTE_MINSC - sc.min_score(L) if byte_range else 0)
        probs, meta = _fit_512(reads, quals, probs, meta)
        c1 = probs["tidx"] == 1
        assert (c1 & (probs["refl"] == 0)).any() and (c1 & (probs["refr"] == len(mate_genome[1]) - 1)).any()   # windows cut at the ends
        assert ((probs["tidx"] == 0) & (probs["refl"] <= NGAP_AT) & (probs["refr"] >= NGAP_AT)).any()         # and over the N gap
        return reads, quals, probs, meta
    keys, _ = _four_calls(gpu, R, mate_genome, make)
    assert [k[0] for k in keys] == [1, 0, 3, 1], keys


@pytest.mark.parametrize("L", [257, 384, 512])
def test_long_local_matches_reference(gpu, synth_index, synth_genome, L):
    """--local reads with junk ends (soft clipping) whose scores pass 255: the reference reruns them in its i16 matrix"""
    gpu.load_index_files(synth_index)
    gpu.set_scoring(local=True)
    R = Reference(synth_index)
    sc = policy.Scoring.default(True)
    reads, quals, truth = synth.make_reads(synth_genome, 60, L, seed=3 * L, sub_rate=0.01, indel_rate=0.003, random_frac=0.05)
    rng = np.random.default_rng(L + 1)
    for i, r in enumerate(reads):
        if i % 3 == 0:
            k = int(rng.integers(3, L // 5))
            r[:k] = rng.integers(0, 4, k)
        if i % 4 == 0:
            k = int(rng.integers(3, L // 5))
            r[-k:] = rng.integers(0, 4, k)
        if i % 7 == 0:
            r[rng.integers(0, L)] = 4
    probs, meta = _problems(synth_genome, reads, truth, sc, rng)
    try:
        key, (nfound, naln, _) = _run(gpu, R, synth_genome, reads, quals, probs, meta, 3, local=True)
    finally:
        gpu.set_scoring(local=False)
    assert key == ("local", 16)
    assert nfound > 30 and naln > 30


@pytest.mark.parametrize("L", [300, 424, 512])
@pytest.mark.parametrize("kind", ["mode1", "mode3", "local"])
def test_long_candidate_fates_match_the_oracle_attempt_log(gpu, synth_index, synth_genome, L, kind):
    """FAILED / SUCCEEDED exactly at the candidates the reference starts a backtrace from, in order: each such attempt is an RNG
    reseed of the engine, so the fates of long reads decide its later draws"""
    from oracle_lib import Oracle, oracle_dp
    local = kind == "local"
    gpu.load_index_files(synth_index)
    gpu.set_scoring(local=local)
    gpu.set_dp_mode(1 if kind == "mode1" else 3)
    O = Oracle(synth_index)
    sc = policy.Scoring.default(local)
    reads, quals, truth = synth.make_reads(synth_genome, 60, L, seed=91 + L, sub_rate=0.02, indel_rate=0.006)
    probs = np.zeros(len(reads), dtype=DP_PROBLEM)
    meta = []
    for i, r in enumerate(reads):
        c, pos, fw = int(truth[i][0]), int(truth[i][1]), int(truth[i][2]) > 0
        if c < 0:
            c, pos, fw = 0, 1000 + i, True
        minsc = max(sc.min_score(L), BYTE_MINSC) if kind == "mode3" else sc.min_score(L)
        tlen = len(synth_genome[c])
        found, rect = policy.frame_seed_extension_rect(pos, L, tlen, sc.max_read_gaps(minsc, L), sc.max_ref_gaps(minsc, L), sc.n_ceil(L))
        probs[i] = (i, int(fw), c, rect.refl, rect.refr, rect.triml, rect.corel, rect.corer, minsc, sc.n_ceil_raw(L), 0)
        meta.append(rect)
    if not local:
        assert _mode(int(probs["minsc"].min()), 1 if kind == "mode1" else 3) == (1 if kind == "mode1" else 3)
    try:
        summ, cands, alns, ops = gpu.dp_extend(ReadBatch.from_list(reads, quals), probs, max_cands=32768 if local else 2048, max_alns=32)
    finally:
        gpu.set_dp_mode(3)
        gpu.set_scoring(local=False)
    n_att = 0
    for i, r in enumerate(reads):
        assert summ[i]["flags"] == 0, (i, summ[i])
        d = oracle_dp(O, local, r, quals[i], bool(probs[i]["fw"]), int(probs[i]["tidx"]), meta[i], int(probs[i]["minsc"]),
                      int(probs[i]["nceil"]), max_cands=65536, max_alns=64, max_edits=16384, attempts=True)
        assert bool(summ[i]["found"]) == bool(d["found"]), i
        if not d["found"]:
            continue
        got = [(ci, int(cands[i][ci]["fate"])) for ci in range(int(summ[i]["ncand"])) if int(cands[i][ci]["fate"]) in (2, 3)]
        want = [(ci, 3 if ai >= 0 else 2) for (s, ai), ci in zip(d["attempts"], d["attempt_cands"])]
        assert got == want, (i, got[:6], want[:6])
        n_att += len(want)
    assert n_att > 30


WIDTHS = [1000, 3000, 4000, 4100, 4200, 6000, 8000, 16000]     # (16000: bt2g_dp_extend takes up to 16384 columns)


def _wide_problems(genome, L, W, sc, rng, byte_range):
    """mate windows of W columns (frameFindMateRect around an anchor whose mate may lie anywhere in a span of about W - L columns,
    as under -X of about W): the true mate somewhere inside, a random read, windows over the tandem family, over the N gap and off
    both ends of the contig"""
    c, tlen = 0, len(genome[0])
    reads, quals, probs, meta = [], [], [], []
    starts = [int(x) for x in rng.integers(0, tlen - W, 6)] + [TANDEM_AT - W // 2, NGAP_AT - W // 3, -40, tlen - W + 40]
    for k, s in enumerate(starts):
        r = rng.integers(0, 4, L).astype(np.uint8)
        fw = bool(rng.integers(0, 2))
        if k != 1:
            ms = min(max(s + int(rng.integers(0, W - L)), 0), tlen - L)
            if k == 6:
                ms = TANDEM_AT + int(rng.integers(-5, 6))
            r = genome[c][ms:ms + L].copy()
            r[r > 3] = int(rng.integers(0, 4))
            r = _mutate(rng, r, int(rng.integers(0, 4)))
            if not fw:
                r = synth.revcomp(r)
        minsc = max(sc.min_score(L), BYTE_MINSC) if byte_range else sc.min_score(L)
        rdg, rfg = sc.max_read_gaps(minsc, L), sc.max_ref_gaps(minsc, L)
        big = 1 << 30
        _, r0 = policy.frame_find_mate_rect(True, big, big, big, big, L, 1 << 40, rdg, rfg, sc.n_ceil(L))
        span = W - (r0.refr - r0.refl + 1)                                 # rr - rl that makes the window W columns wide
        rl = s + big - r0.refl                                             # and start at s (cut to the contig there)
        found, rect = policy.frame_find_mate_rect(True, rl, rl, rl, rl + span, L, tlen, rdg, rfg, sc.n_ceil(L))
        assert found
        probs.append((len(reads), int(fw), c, rect.refl, rect.refr, rect.triml, rect.corel, rect.corer, minsc, sc.n_ceil_raw(L), 0))
        meta.append((tlen, rect, minsc))
        reads.append(r)
        quals.append(rng.integers(35, 74, L).astype(np.uint8))
    return reads, quals, np.array(probs, dtype=DP_PROBLEM), meta


@pytest.mark.parametrize("L", [150, 300])
@pytest.mark.parametrize("kind", ["mode1", "mode3", "local"])
def test_wide_mate_windows_match_reference(gpu, mate_index, mate_genome, L, kind):
    """windows up to 8000 columns (the widest mate window the device engine frames) and 16000 (the coroutine engine's windows under
    larger -X): 4000-4200 straddle the width from which 4 warps of k_dp_e2e_x2 or 8 of k_dp_tail_h no longer fit one
    block's shared memory; each kernel takes fewer warps per block there, and the answers stay the reference's"""
    local = kind == "local"
    gpu.load_index_files(mate_index)
    gpu.set_scoring(local=local)
    R = Reference(mate_index)
    sc = policy.Scoring.default(local)
    cap = {"mode1": 1, "mode3": 3, "local": 3}[kind]       # (a 150 bp read's default minsc already fits a byte)
    rng = np.random.default_rng(L + len(kind))
    fits = []
    try:
        for W in WIDTHS:
            reads, quals, probs, meta = _wide_problems(mate_genome, L, W, sc, rng, kind == "mode3")
            assert int((probs["refr"] - probs["refl"] + 1).max()) == W
            key, (nfound, naln, _) = _run(gpu, R, mate_genome, reads, quals, probs, meta, cap, local=local)
            assert key[0] == ("local" if local else int(kind[-1])), key
            assert nfound >= 5 and naln >= 5, (W, nfound, naln)
            fits.append(_fits_four_warps(W, 0 if local else key[0], key[1]))
    finally:
        gpu.set_scoring(local=False)
    if local:
        assert fits == [W < 8192 for W in WIDTHS], fits                  # local blocks of 4 warps fit up to about 8300 columns
    else:
        # the limit lies between 3000 and 4200 columns (3990 for the tail at R = 10, 4058 at R = 5, 4145 for 4 warps of the
        # s16x2 kernels): the widths below it run at the old block shapes, the ones above on fewer warps per block
        assert fits == sorted(fits, reverse=True) and fits.index(False) in (2, 3, 4), fits


def test_zz_every_long_kernel_instantiation_ran():
    """the end of the file: every kernel generation and rows-per-lane instantiation that reads of 251-512 bases reach ran with found
    alignments above"""
    want = {(0, 16), (1, 8), (1, 16), (3, 10), (3, 12), (3, 16), ("local", 16)}
    assert want <= RAN, sorted(want - RAN, key=str)
