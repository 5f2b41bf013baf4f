"""How deep the live band of a mate-finding rectangle reaches: how many rows the top row block of the end-to-end DP fill
(k_dp_fill_h, DESIGN.md sections 3 and 9) sweeps at full width to no purpose.

Pairs come from bench.py's generator (make_genome_gpu / make_pairs_gpu, run on the CPU over a scaled-down genome).  Mate 1 is
placed by an exact 20-mer lookup; its mate window is framed as the engine frames it (PairedEndPolicy.other_mate,
frame_find_mate_rect), and mate 2 is filled end to end over that window with the default scoring (quality-aware mismatch
penalty, N penalty, gaps 5+3, gap barrier 4) at the workload's minimum score.  A cell is live when its best path scores at
least minsc.  A true mate keeps a narrow band live down to the last row; what sizes the top block is how deep the rest of the
window stays live.  The script prints, per rectangle, the deepest row in which more than 15 % of the columns (a true mate band covers about 8 %) are live, and the
share of live cells per row.

    python tools/dp_live_rows.py [--pairs 2000] [--len 150] [--genome-mbp 4]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NEG = -(1 << 20)


def fill_live(reads, quals, refs, minsc, sc):
    """End-to-end fill of a batch of equal-length reads against equal-width windows; live[b, i] = the share of row i of window b
    whose cells score >= minsc.  Clamping below minsc is exact here: every increment is <= 0 with no match bonus."""
    nb, L = reads.shape
    W = refs.shape[1]
    mmp = np.array([[sc.mm_penalty(int(q)) for q in row] for row in quals])
    rdo, rde, rfo, rfe = sc.read_gap_open(), sc.read_gap_extend(), sc.ref_gap_open(), sc.ref_gap_extend()
    H = np.full((nb, W), NEG)
    F = np.full((nb, W), NEG)
    live = np.zeros((nb, L))
    for i in range(L):
        rc = reads[:, i:i + 1]
        nmask = (rc > 3) | (refs > 3)
        s = np.where(nmask, -sc.n_pen, np.where(rc == refs, 0, -mmp[:, i:i + 1]))
        bar = i < sc.gapbar or L - 1 - i < sc.gapbar
        if i == 0:
            Hn = s.copy()
            Fn = np.full((nb, W), NEG)
        else:
            Hd = np.concatenate([np.full((nb, 1), NEG), H[:, :-1]], axis=1) + s
            Fn = np.full((nb, W), NEG) if bar else np.maximum(H - rfo, F - rfe)
            Hn = np.maximum(Hd, Fn)
        if not bar:
            E = np.full(nb, NEG)
            for j in range(W):
                Hn[:, j] = np.maximum(Hn[:, j], E)
                E = np.maximum(Hn[:, j] - rdo, E - rde)
        Hn = np.where(Hn < minsc, NEG, Hn)
        Fn = np.where(Fn < minsc, NEG, Fn)
        H, F = Hn, Fn
        live[:, i] = (H > NEG).mean(axis=1)
    return live


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2000)
    ap.add_argument("--len", type=int, default=150)
    ap.add_argument("--genome-mbp", type=float, default=4.0)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    import torch
    import bench
    from bowtie2_b200 import policy
    dev = torch.device("cpu")
    clen = int(args.genome_mbp * 1e6 / 2)
    contigs = bench.make_genome_gpu(torch, dev, 2, clen)
    reads, quals = bench.make_pairs_gpu(torch, dev, contigs, args.pairs, args.len, seed=args.seed)
    genome = [c.numpy() for c in contigs]
    reads, quals = reads.numpy(), quals.numpy() - 33
    K = 20
    index = {}
    for ci, g in enumerate(genome):
        for p in range(0, len(g) - K):
            index.setdefault(g[p:p + K].tobytes(), (ci, p))
    comp = np.array([3, 2, 1, 0, 4], np.uint8)
    sc = policy.Scoring.default(False)
    pe = policy.PairedEndPolicy()
    L = args.len
    minsc = sc.min_score(L)
    groups = {}                                     # window width -> list of (read, quals, window)
    for k in range(args.pairs):
        m1, m2, q2 = reads[2 * k], reads[2 * k + 1], quals[2 * k + 1]
        hit = None
        for fw, r in ((True, m1), (False, comp[m1[::-1]])):
            for o in (0, 40, 80, L - K):
                h = index.get(r[o:o + K].tobytes())
                if h is not None:
                    hit = (h[0], h[1] - o, fw)
                    break
            if hit:
                break
        if hit is None:
            continue
        c, off, fw = hit
        tlen = len(genome[c])
        om = pe.other_mate(True, fw, off, -1, tlen, L, L)
        if om is None:
            continue
        oleft, oll, olr, orl, orr, ofw = om
        found, rect = policy.frame_find_mate_rect(not oleft, oll, olr, orl, orr, L, tlen, sc.max_read_gaps(minsc, L),
                                                  sc.max_ref_gaps(minsc, L), sc.n_ceil(L))
        if not found:
            continue
        ref = np.full(rect.refr - rect.refl + 1, 4, np.uint8)
        lo, hi = max(rect.refl, 0), min(rect.refr + 1, tlen)
        ref[lo - rect.refl:hi - rect.refl] = genome[c][lo:hi]
        rd, qd = (m2, q2) if ofw else (comp[m2[::-1]], q2[::-1])
        groups.setdefault(len(ref), []).append((rd, qd, ref))
    deepest, rows = [], []
    for W, items in groups.items():
        live = fill_live(np.stack([x[0] for x in items]).astype(np.int64), np.stack([x[1] for x in items]),
                         np.stack([x[2] for x in items]).astype(np.int64), minsc, sc)
        rows.append(live)
        deepest += [int(np.nonzero(r > 0.15)[0].max()) if (r > 0.15).any() else -1 for r in live]
    live = np.concatenate(rows)
    d = np.array(deepest)
    print(f"{len(d)} mate rectangles of {args.pairs} pairs, read length {L}, minsc {minsc}, widths {min(groups)}..{max(groups)}")
    print("deepest row with > 15 %% of its cells live: min %d, median %d, 99th percentile %d, max %d"
          % (d.min(), np.median(d), np.percentile(d, 99), d.max()))
    for t in (31, 47, 63):
        print(f"  rectangles with such a row below row {t}: {np.mean(d > t) * 100:.2f} %")
    print("live cells per row: " + " ".join(f"{i}:{live[:, i].mean() * 100:.1f}%" for i in range(0, L, 4) if i < 72))
    print(f"live cells in rows 0-47: {live[:, :48].mean() * 100:.1f} %, rows 48-63: {live[:, 48:64].mean() * 100:.2f} %, "
          f"rows 32-63: {live[:, 32:64].mean() * 100:.2f} %")


if __name__ == "__main__":
    main()
