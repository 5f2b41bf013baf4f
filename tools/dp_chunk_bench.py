"""How the chunking of the split end-to-end DP (mode 3: k_dp_fill_h + k_dp_tail_h over chunks of problems) shows in the device
engine's DP times.

A seeded synthetic genome with repeat families (bench.py's generator) is indexed on the GPU (bowtie2_b200.index_build); one and
then two XEngines align 2x150 bp FR pairs with --very-sensitive (bench.py's default workload at a smaller genome).  The DP
workspace budget (BT2G_DP_CHUNK_MB, read when an engine is created) is swept so that it holds 1.0, 2.0, 2.18 (the default
3 GiB) and 3.0 resident rounds of the mate fill: one round is the problems the fill keeps resident on the whole GPU (two per warp,
4 warps per block, 8 blocks per SM at the default mate window).  Per setting: wall ms per batch, and the engines' stage_ms of the
fill and the tail (summed over the engines, per batch).  One run with BT2G_XE_DEBUG gives the per-wave anchor / mate problem counts.
Prints one JSON line; a table on stderr.

usage: python tools/dp_chunk_bench.py [--genome-mbp 300] [--pairs 250000] [--steps 3] [--rounds 1.0,2.0,2.18,3.0]"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": q[0], "power_limit_w": float(q[1]), "sm_clock_mhz": int(q[2]), "sm_clock_max_mhz": int(q[3])}
    except Exception as e:                                    # (no nvidia-smi: the number still stands, without its conditions)
        return {"error": str(e)}


def code_stride_mode3(max_col, max_len):
    """dp_code_stride (dp_device.cuh) for mode 3: rows per lane rounded up to whole 2-row blocks, maxCol + 36 steps, 256 B aligned"""
    r = next(x for x in (4, 5, 6, 8, 10, 12, 16) if 32 * x >= max_len)
    r = (r + 1) // 2 * 2
    return ((max_col + 36) * 32 * r + 255) & ~255


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome-mbp", type=float, default=300.0)
    ap.add_argument("--pairs", type=int, default=250_000, help="pairs per engine and batch")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", default="1.0,2.0,2.18,3.0", help="mate fill rounds per workspace budget")
    args = ap.parse_args()
    import torch
    import bench
    from bowtie2_b200 import Bt2Gpu
    from bowtie2_b200.index_build import build_index
    from bowtie2_b200.lib import XEngine, policy_params
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    t0 = time.time()
    n_contigs = 4
    contigs = bench.make_genome_gpu(torch, dev, n_contigs, int(args.genome_mbp * 1e6 / n_contigs))
    built = build_index(contigs, off_size=4)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    L = 150
    E2 = 2
    reads, quals = bench.make_pairs_gpu(torch, dev, contigs, E2 * args.pairs * (args.steps + 1), L, seed=3)
    del contigs
    gpu = Bt2Gpu(0)
    gpu.load_index_device(built.device_desc(dev), keep=built)
    offs = torch.arange(0, reads.shape[0] * L + 1, L, dtype=torch.int64, device=dev)
    reads, quals = reads.contiguous(), quals.contiguous()
    print(f"[dp_chunk_bench] genome + index + reads in {time.time() - t0:.0f} s", file=sys.stderr, flush=True)
    prm = policy_params("very-sensitive", paired=True, seed=0)

    # the mate window of XEngine at the default settings (xengine.cu createEngine): maxfrag + 2 maxLen + 2 gapMax + 16, + 1
    max_col_m = 500 + 2 * L + 2 * 29 + 16 + 1
    stride_m = code_stride_mode3(max_col_m, L)
    resident = 2 * 4 * 8 * sms                                # problems the mate fill holds at once

    def part(j, i):                                           # engine j's part of batch i (device pointers)
        lo = (i * E2 + j) * args.pairs * 2
        return reads[lo:].data_ptr(), quals[lo:].data_ptr(), offs.data_ptr(), 2 * args.pairs

    def run(n_eng, budget_mb):
        if budget_mb:
            os.environ["BT2G_DP_CHUNK_MB"] = str(budget_mb)
        else:
            os.environ.pop("BT2G_DP_CHUNK_MB", None)
        engines = [XEngine(gpu, prm, args.pairs, L) for _ in range(n_eng)]
        os.environ.pop("BT2G_DP_CHUNK_MB", None)
        for j, e in enumerate(engines):                      # warm-up
            s, q, o, n = part(j, 0)
            e.run_dev(s, q, o, n)
        torch.cuda.synchronize()
        tb = [0.0]
        acc = {"dp_fill": 0.0, "dp_tail": 0.0, "mate_dp": 0.0, "seed_dp": 0.0, "total": 0.0}
        stats = {"mate_dps": 0, "seed_dps": 0, "waves": 0}
        lock = threading.Lock()

        def work(j):
            torch.cuda.set_device(dev)
            time.sleep(tb[0] * j / n_eng)                     # out of phase, as bench.py starts its engines
            for i in range(1, args.steps + 1):
                s, q, o, n = part(j, i)
                st = engines[j].run_dev(s, q, o, n)
                sm = engines[j].stage_ms()
                with lock:
                    for k in acc:
                        acc[k] += sm[k]
                    for k in stats:
                        stats[k] += st[k]
        s0 = time.perf_counter()
        s, q, o, n = part(0, 1)
        engines[0].run_dev(s, q, o, n)
        tb[0] = time.perf_counter() - s0                       # one batch of one engine
        w0 = time.perf_counter()
        th = [threading.Thread(target=work, args=(j,)) for j in range(n_eng)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - w0) / args.steps
        for e in engines:
            e.close()
        torch.cuda.empty_cache()
        per = {k: round(v / args.steps, 2) for k, v in acc.items()}
        return {"engines": n_eng, "budget_mb": budget_mb, "wall_ms_per_batch": round(wall * 1e3, 1), "stage_ms": per,
                "mate_dps_per_batch": stats["mate_dps"] // args.steps, "seed_dps_per_batch": stats["seed_dps"] // args.steps}

    # per-wave queue sizes: one batch of one engine with BT2G_XE_DEBUG (the engine's per-wave log on stderr)
    os.environ["BT2G_XE_DEBUG"] = "1"
    eng = XEngine(gpu, prm, args.pairs, L)
    os.environ.pop("BT2G_XE_DEBUG", None)
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            s, q, o, n = part(0, 0)
            eng.run_dev(s, q, o, n)
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        waves = [(int(a), int(b)) for a, b in re.findall(r"dpA (\d+) dpM (\d+)", f.read())]
    eng.close()
    torch.cuda.empty_cache()

    out = {"metric": "split end-to-end DP chunking", "genome_mbp": args.genome_mbp, "pairs_per_engine": args.pairs, "card": card(),
           "mate_code_stride": stride_m, "mate_fill_resident_problems": resident,
           "waves_dpA_dpM": waves, "runs": []}
    rounds = [float(x) for x in args.rounds.split(",")]
    for n_eng in (1, 2):
        for r in rounds:
            mb = int(r * resident * stride_m) >> 20
            res = run(n_eng, mb)
            res["mate_rounds_per_budget"] = r
            out["runs"].append(res)
            print(f"[dp_chunk_bench] {json.dumps(res)}", file=sys.stderr, flush=True)
    out["card_after"] = card()
    print(f"{'eng':>3} {'rounds':>6} {'MB':>6} {'wall ms':>8} {'fill':>7} {'tail':>7} {'mateDP':>7} {'seedDP':>7}", file=sys.stderr)
    for r in out["runs"]:
        s = r["stage_ms"]
        print(f"{r['engines']:>3} {r['mate_rounds_per_budget']:>6} {r['budget_mb']:>6} {r['wall_ms_per_batch']:>8} {s['dp_fill']:>7} {s['dp_tail']:>7} "
              f"{s['mate_dp']:>7} {s['seed_dp']:>7}", file=sys.stderr)
    gpu.close()
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
