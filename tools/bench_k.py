"""-k / -a throughput of the device engine (bt2g_xengine_create_k / _align_k) against the coroutine engine that served -k before it
(bt2g_policy_align_pairs_k / _k over bt2g_policy_backend_gpu), with the -M device engine for context.

A seeded synthetic genome with repeat families (bench.py's generator) is indexed on the GPU (bowtie2_b200.index_build), then:
  * 2x150 bp FR pairs, --very-sensitive -k 5, and 150 bp unpaired reads, --sensitive -k 10;
  * per workload the three paths run on the same batch, alternating, after a warm-up; the coroutine engine runs on a smaller sample
    (the first `--slow-units` units of the batch) and its rate is per unit of that sample;
  * the device engine's entry arrays must equal the coroutine engine's on that shared sample (every written row).
Prints one JSON line: units/s per path and workload, fallback units, and the card's name, power limit and SM clock read in the same run.

usage: python tools/bench_k.py [--genome-mbp 300] [--pairs 200000] [--reads 200000] [--slow-units 4000] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": q[0], "power_limit_w": float(q[1]), "sm_clock_mhz": int(q[2]), "sm_clock_max_mhz": int(q[3])}
    except Exception as e:                                    # (no nvidia-smi: the number still stands, without its conditions)
        return {"error": str(e)}


def equal_entries(paired, a, b):
    """entry arrays (res, ops, pairs, n_entries) of two engines equal on every written row"""
    res_a, ops_a, pairs_a, cnt_a = a
    res_b, ops_b, pairs_b, cnt_b = b
    if not np.array_equal(cnt_a, cnt_b):
        return False
    per = np.maximum(cnt_a.astype(np.int64), 1)
    u = np.repeat(np.arange(len(per)), per)
    e = np.arange(len(u)) - np.repeat(np.cumsum(per) - per, per)
    ra, rb = res_a[u, e], res_b[u, e]
    if ra.tobytes() != rb.tobytes():
        return False
    if paired and pairs_a[u, e].tobytes() != pairs_b[u, e].tobytes():
        return False
    oa, ob = ops_a[u, e].reshape(ra.size, -1), ops_b[u, e].reshape(rb.size, -1)
    w = min(oa.shape[1], ob.shape[1])
    mask = np.arange(w)[None, :] < np.minimum(ra.reshape(-1)["nops"], w)[:, None]
    return bool(np.array_equal(np.where(mask, oa[:, :w], 0), np.where(mask, ob[:, :w], 0)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome-mbp", type=float, default=300.0)
    ap.add_argument("--pairs", type=int, default=200_000)
    ap.add_argument("--reads", type=int, default=200_000)
    ap.add_argument("--slow-units", type=int, default=4000)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    import bench
    from bowtie2_b200 import Bt2Gpu
    from bowtie2_b200.index_build import build_index
    from bowtie2_b200.lib import ReadBatch, XEngine, policy_align_k, policy_align_pairs_k, policy_backend_gpu, policy_params
    dev = torch.device("cuda", 0)
    t0 = time.time()
    n_contigs = 4
    contigs = bench.make_genome_gpu(torch, dev, n_contigs, int(args.genome_mbp * 1e6 / n_contigs))
    built = build_index(contigs, off_size=4)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    pr, pq = bench.make_pairs_gpu(torch, dev, contigs, args.pairs, 150, seed=3)
    ur, uq = bench.make_reads_gpu(torch, dev, contigs, args.reads, 150, seed=4)
    del contigs
    gpu = Bt2Gpu(0)
    gpu.load_index_device(built.device_desc(dev), keep=built)
    print(f"[bench_k] genome + index + reads in {time.time() - t0:.0f} s", file=sys.stderr, flush=True)

    def batch_of(r, q):
        r, q = r.cpu().numpy(), q.cpu().numpy()
        n, L = r.shape
        return ReadBatch(np.ascontiguousarray(r.reshape(-1)), np.arange(0, (n + 1) * L, L, dtype=np.uint64), np.ascontiguousarray(q.reshape(-1)))

    out = {"metric": "-k throughput, device engine vs coroutine engine", "genome_mbp": args.genome_mbp, "card": card(), "workloads": {}}
    for name, paired, preset, k, r, q, n in (("pe150_very_sensitive_k5", True, "very-sensitive", 5, pr, pq, args.pairs),
                                           ("se150_sensitive_k10", False, "sensitive", 10, ur, uq, args.reads)):
        batch = batch_of(r, q)
        slow = batch_of(r[:args.slow_units * (2 if paired else 1)], q[:args.slow_units * (2 if paired else 1)])
        cap = 2 * k + 2 if paired else k
        prm_k = policy_params(preset, paired=paired, k=k, host_threads=8)
        prm_m = policy_params(preset, paired=paired, host_threads=8)
        ek = XEngine(gpu, prm_k, n, 150, max_per_unit=cap)
        em = XEngine(gpu, prm_m, n, 150)
        be = policy_backend_gpu(gpu)

        names_all = [f"r{i // 2 if paired else i}" for i in range(batch.n)]
        names_slow = names_all[:slow.n]

        def coroutine(b):
            gpu.set_scoring(local=False)
            return (policy_align_pairs_k if paired else policy_align_k)(gpu._lib, be, prm_k, b, names_slow, cap)
        # warm-up (and the identity check on the shared sample)
        dk = ek.align_k(slow, names_slow)
        ck = coroutine(slow)
        same = equal_entries(paired, dk[:4], (ck[0], ck[1], ck[2], ck[3]) if paired else (ck[0], ck[1], None, ck[2]))
        ek.align_k(batch, names_all)
        em.align(batch, names_all)
        t = {"device_k": [], "coroutine_k": [], "device_m": []}
        fb = 0
        for _ in range(args.rounds):                          # alternating paths
            s = time.perf_counter(); got = ek.align_k(batch, names_all); t["device_k"].append(time.perf_counter() - s)
            fb = got[5]["fallback_units"]
            s = time.perf_counter(); coroutine(slow); t["coroutine_k"].append(time.perf_counter() - s)
            s = time.perf_counter(); em.align(batch, names_all); t["device_m"].append(time.perf_counter() - s)
        ek.close(); em.close()
        unit = "pairs" if paired else "reads"
        out["workloads"][name] = {
            "units": n, "unit": unit, "coroutine_sample_units": args.slow_units, "identical_on_sample": same, "device_k_fallback_units": int(fb),
            f"device_k_{unit}_per_s": [round(n / x) for x in t["device_k"]],
            f"coroutine_k_{unit}_per_s": [round(args.slow_units / x) for x in t["coroutine_k"]],
            f"device_m_{unit}_per_s": [round(n / x) for x in t["device_m"]],
        }
        print(f"[bench_k] {name}: {json.dumps(out['workloads'][name])}", file=sys.stderr, flush=True)
    out["card_after"] = card()
    gpu.close()
    print(json.dumps(out))
    return 0 if all(w["identical_on_sample"] for w in out["workloads"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
