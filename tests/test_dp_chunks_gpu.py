"""GPU: the split end-to-end DP (k_dp_fill_h + k_dp_tail_h) gives the same answers however a queue is cut into chunks.

A queue runs as ceil(n / capacity) chunks of equal size (dp_chunk_size), each kernel hands out its chunk's problems through an
atomic counter, and the device engine alternates consecutive chunks between its two streams and the two halves of its workspace.
So which warp takes which problem, and where a problem's bytes sit, change with the workspace budget (BT2G_DP_CHUNK_MB, read per
bt2g_dp_extend call and per engine); summaries, candidates with their fates, alignments and op strings must not."""
import numpy as np
import pytest

from bowtie2_b200 import policy
from bowtie2_b200.lib import ReadBatch
from oracle_lib import Reference, have_reference
from test_dp_block_edges_gpu import _assert_same
from test_dp_gpu import _check
from test_dp_mate_gpu import _mate_problems, mate_genome, mate_index  # noqa: F401  (fixtures)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

L = 150


def _stride(probs, reads):
    """dp_code_stride (dp_device.cuh) of a bt2g_dp_extend call in mode 3"""
    max_col = int((probs["refr"] - probs["refl"] + 1).max()) + 1
    r = next(x for x in (4, 5, 6, 8, 10, 12, 16) if 32 * x >= max(len(x) for x in reads))
    r = (r + 1) // 2 * 2
    return ((max_col + 36) * 32 * r + 255) & ~255


def _extend(gpu, batch, probs, monkeypatch, budget_mb):
    monkeypatch.setenv("BT2G_DP_CHUNK_MB", str(budget_mb))
    return gpu.dp_extend(batch, probs, max_cands=256, max_alns=8, max_ops=L + 80)


@pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")
def test_dp_chunks_same_as_one_chunk(gpu, mate_index, mate_genome, monkeypatch):
    """Mate rectangles repeated into queues of up to 7 x 8448 problems: budgets that cut one call into 1, 2, 3 and 7 chunks, with
    counts at the chunk capacity and at the fill's resident rounds (two problems per warp, 32 warps per SM) plus or minus one;
    every copy of a problem answers as the problem itself, which matches the reference SwAligner."""
    import torch
    gpu.load_index_files(mate_index)
    gpu.set_scoring(local=False)
    R = Reference(mate_index)
    sc = policy.Scoring.default(False)
    rng = np.random.default_rng(150)
    reads, quals, base, meta = _mate_problems(mate_genome, L, sc, rng)
    monkeypatch.setenv("BT2G_DP_CHUNK_MB", "1")
    nfound, naln, _ = _check(gpu, R, mate_genome, reads, quals, base, meta)
    assert nfound > 20 and naln > 20
    batch = ReadBatch.from_list(reads, quals)
    want = _extend(gpu, batch, base, monkeypatch, 4096)
    stride = _stride(base, reads)
    rnd = 64 * torch.cuda.get_device_properties(0).multi_processor_count
    cap_small = 1024                                                         # the workspace floor: BT2G_DP_CHUNK_MB=1
    mb_round = -(-rnd * stride // (1 << 20))                                 # one resident round (a few problems more)
    cap_round = mb_round * (1 << 20) // stride
    cases = [(cap_small, 1, 1024), (cap_small, 1, 1025), (cap_small, 1, 2049), (cap_small, 1, 7167),
             (cap_round, mb_round, rnd - 1), (cap_round, mb_round, rnd + 1), (cap_round, mb_round, 2 * rnd + 1),
             (cap_round, mb_round, 7 * rnd - 1)]
    chunks = set()
    for cap, mb, n in cases:
        idx = rng.integers(0, len(base), n)
        probs = base[idx]
        got = _extend(gpu, batch, probs, monkeypatch, mb)
        one = _extend(gpu, batch, probs, monkeypatch, -(-n * stride // (1 << 20)) + 1)     # the whole queue in one chunk
        _assert_same(got, one)
        _assert_same(got, tuple(x[idx] for x in want))
        chunks.add(-(-n // cap))
    assert {1, 2, 3, 7} <= chunks, chunks


def test_xengine_small_chunks_same_results(tmp_path, monkeypatch):
    """A paired --very-sensitive engine whose DP queues run as many small chunks, alternating between its two streams (the
    side-by-side launches of small waves turned off), leaves the same result arrays as an engine with the default workspace."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from bowtie2_b200 import Bt2Gpu, synth
    from bowtie2_b200.lib import XEngine, policy_params
    from oracle_lib import ref_bin
    if not have_reference():
        pytest.skip("oracle/_ref not built")
    import subprocess
    genome = synth.make_genome(n_contigs=3, contig_len=200000, seed=17, repeat_frac=0.2, repeat_len=400, repeat_copies=150, n_gap=53)
    fa, base = str(tmp_path / "g.fa"), str(tmp_path / "g")
    synth.write_fasta(fa, genome)
    subprocess.check_call([ref_bin("bowtie2-build-s"), "--seed", "0", "--quiet", fa, base])
    n = 6000
    reads, quals, _ = synth.make_pairs(genome, n, L, seed=43, sub_rate=0.01, indel_rate=0.001, ins_mean=350, ins_sd=40)
    g = Bt2Gpu(0)
    g.load_index_files(base)
    batch = ReadBatch.from_list(reads, quals)
    prm = policy_params("very-sensitive", paired=True)
    out = []
    for env in ({}, {"BT2G_DP_CHUNK_MB": "1", "BT2G_XE_DP_SERIAL": "1"}):
        for k in ("BT2G_DP_CHUNK_MB", "BT2G_XE_DP_SERIAL"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng = XEngine(g, prm, n, L)
        try:
            res, ops, pairs, stats = eng.align(batch)
            ops = np.where(np.arange(ops.shape[1])[None, :] < res["nops"][:, None], ops, 0)      # (bytes past nops are not written)
            out.append((res.tobytes(), ops.tobytes(), pairs.tobytes(), stats))
        finally:
            eng.close()
    assert out[0][3]["mate_dps"] > 2048, out[0][3]                          # more than two chunks of 1024 in the small engine
    assert out[0][:3] == out[1][:3]
    g.close()
