"""Parity fuzz on the CPU: the device engine's state machine (csrc/xengine.cuh, the code k_xe_step runs) driven on the host over the
oracle-backed entry-point table (bt2g_xengine_align_host), against the UNMODIFIED reference program (oracle/_ref/bowtie2-align-s) on
fresh synthetic genomes and reads: presets x end-to-end / local x unpaired / paired x read lengths x error rates x the policy options
the engines take (--nofw/--norc, -L, -D, -R, -i, --ff/--rf, -I/-X, --dovetail, --no-contain, --no-overlap, --no-mixed,
--no-discordant, --mp, --np, --rdg, --rfg, --ma, --score-min, --n-ceil, --seed, -M; .bt2 and .bt2l indexes).  Every SAM record must be identical.

Test infrastructure (uses oracle/): `python tests/parity_fuzz.py SEED CASES` prints one line per case and a JSON summary;
tests/test_parity_fuzz.py runs a few fixed seeds.  With --device (a GPU) the same cases run on the device engine itself
(bt2g_xengine_align / _align_k over the CUDA kernels); tests/test_xengine_fuzz_gpu.py runs a fixed list of them."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

REF = os.path.join(ROOT, "oracle", "_ref", "bowtie2-align-s")


def draw_case(seed, k):
    """configuration k of run `seed`: genome, reads, preset and options (as keyword arguments of lib.policy_params + the reference's
    flags).  Every group of choices has its own generator, so that a new group does not move the cases of the existing seeds."""
    from bowtie2_b200 import policy
    rng = np.random.default_rng([seed, k, 0])
    c = {"genome_seed": int(rng.integers(1, 1 << 30)), "n_contigs": int(rng.integers(1, 4)), "contig_len": int(rng.integers(8000, 30000)),
         "repeat_frac": float(rng.choice([0.02, 0.1, 0.3])), "repeat_len": int(rng.integers(100, 600)), "repeat_copies": int(rng.integers(3, 20)),
         "n_gap": int(rng.integers(0, 60)), "local": bool(rng.integers(0, 2)), "paired": bool(rng.integers(0, 2)),
         "preset": str(rng.choice(["very-fast", "fast", "sensitive", "very-sensitive"])), "read_len": int(rng.choice([30, 50, 75, 100, 150, 250])),
         "sub_rate": float(rng.choice([0.002, 0.01, 0.03, 0.06])), "indel_rate": float(rng.choice([0.0, 0.001, 0.005])),
         "ins_mean": float(rng.choice([250, 350, 450])), "hard_frac": float(rng.choice([0.0, 0.1]))}
    kw, flags = {}, []
    if rng.random() < 0.25:
        if rng.random() < 0.5:
            kw["nofw"] = True; flags.append("--nofw")
        else:
            kw["norc"] = True; flags.append("--norc")
    if rng.random() < 0.3:
        kw["seed_len"] = int(rng.choice([10, 16, 20, 25, 32])); flags += ["-L", str(kw["seed_len"])]
    if rng.random() < 0.3:
        kw["dp_fail_streak"] = int(rng.choice([1, 5, 30])); flags += ["-D", str(kw["dp_fail_streak"])]
    if rng.random() < 0.3:
        kw["seed_rounds"] = int(rng.choice([0, 1, 4])); flags += ["-R", str(kw["seed_rounds"])]
    if rng.random() < 0.3:
        a, b = float(rng.choice([1, 0.5])), float(rng.choice([0.5, 1.15, 2.5]))
        kw["ival"] = policy.SimpleFunc(policy.SIMPLE_FUNC_SQRT, a, b); flags += ["-i", f"S,{a},{b}"]
    if c["paired"]:
        pe = policy.PairedEndPolicy(local=c["local"])
        if rng.random() < 0.3:
            pe.pol = int(rng.choice([policy.PE_POLICY_FF, policy.PE_POLICY_RF])); flags.append("--ff" if pe.pol == policy.PE_POLICY_FF else "--rf")
        if rng.random() < 0.4:
            pe.maxfrag = int(rng.choice([200, 300, 400, 800])); flags += ["-X", str(pe.maxfrag)]
        if rng.random() < 0.3:
            pe.minfrag = int(rng.choice([100, 250, 340])); flags += ["-I", str(pe.minfrag)]
        if rng.random() < 0.2:
            pe.dovetail_ok = True; flags.append("--dovetail")
        if rng.random() < 0.2:
            pe.contain_ok = False; flags.append("--no-contain")
        if rng.random() < 0.2:
            pe.olap_ok = False; flags.append("--no-overlap")
        kw["pe"] = pe
        if rng.random() < 0.25:
            kw["mixed"] = False; flags.append("--no-mixed")
        if rng.random() < 0.25:
            kw["discord"] = False; flags.append("--no-discordant")
    rng = np.random.default_rng([seed, k, 1])                      # scoring options
    if rng.random() < 0.4:
        sc = policy.Scoring.default(c["local"])
        if rng.random() < 0.5:
            mx = int(rng.choice([3, 4, 6, 8])); mn = min(int(rng.choice([1, 2, 3])), mx)
            sc.mmp_max, sc.mmp_min = mx, mn; flags += ["--mp", f"{mx},{mn}"]
        if rng.random() < 0.3:
            sc.n_pen = int(rng.choice([0, 1, 3])); flags += ["--np", str(sc.n_pen)]
        if rng.random() < 0.4:
            sc.rdgap_const, sc.rdgap_linear = int(rng.choice([3, 5, 8])), int(rng.choice([1, 3, 4])); flags += ["--rdg", f"{sc.rdgap_const},{sc.rdgap_linear}"]
        if rng.random() < 0.4:
            sc.rfgap_const, sc.rfgap_linear = int(rng.choice([3, 5, 8])), int(rng.choice([1, 3, 4])); flags += ["--rfg", f"{sc.rfgap_const},{sc.rfgap_linear}"]
        if c["local"] and rng.random() < 0.4:
            sc.match_bonus = int(rng.choice([1, 3])); flags += ["--ma", str(sc.match_bonus)]
        if rng.random() < 0.4:
            if c["local"]:
                a, b = float(rng.choice([1, 10, 20])), float(rng.choice([5.4, 8, 12]))
                sc.score_min_func = policy.SimpleFunc(policy.SIMPLE_FUNC_LOG, a, b); flags += ["--score-min", f"G,{a},{b}"]
            else:
                a, b = float(rng.choice([0, -0.6, -3])), float(rng.choice([-0.3, -0.6, -1.0]))
                sc.score_min_func = policy.SimpleFunc(policy.SIMPLE_FUNC_LINEAR, a, b); flags += ["--score-min", f"L,{a},{b}"]
        if rng.random() < 0.3:
            a, b = float(rng.choice([0, 2])), float(rng.choice([0.05, 0.15, 0.5]))
            sc.n_ceil_over = policy.SimpleFunc(policy.SIMPLE_FUNC_LINEAR, a, b); flags += ["--n-ceil", f"L,{a},{b}"]
        kw["sc"] = sc
    c["large"] = bool(np.random.default_rng([seed, k, 2]).random() < 0.25)          # a .bt2l index (64-bit offsets, 128-byte sides, 64-bit RNG draws) and bowtie2-align-l
    rng = np.random.default_rng([seed, k, 3])                      # the run's RNG seed and -M
    c["run_seed"] = int(rng.choice([0, 0, 1, 7, 12345]))
    if rng.random() < 0.25:
        kw["mhits"] = int(rng.choice([1, 3, 20, 100])); flags += ["-M", str(kw["mhits"])]     # (-M 0 is not an input: bt2_search.cpp:1775 asserts mhits > 0)
    rng = np.random.default_rng([seed, k, 5])                      # -k N / -a: every reported alignment (the coroutine engine: bt2g_policy_align[_pairs]_k)
    u = rng.random()
    if u < 0.25:
        if "mhits" in kw:
            del kw["mhits"]; i = flags.index("-M"); del flags[i:i + 2]      # (-M, -k and -a are mutually exclusive)
        if u < 0.18:
            kw["k"] = int(rng.choice([2, 3, 10])); flags += ["-k", str(kw["k"])]
        else:
            kw["all_hits"] = True; flags.append("-a")
    rng = np.random.default_rng([seed, k, 4])                      # odd reads: ragged lengths (down to 0), Ns, reads across contig ends
    c["ragged"] = bool(rng.random() < 0.3)
    c["n_rate"] = float(rng.choice([0.0, 0.0, 0.02, 0.1]))
    c["straddle"] = bool(rng.random() < 0.3)
    c["read_seed"] = int(rng.integers(1, 1 << 30))
    c["kw"], c["flags"] = kw, flags
    c["dense_sa"], c["seed_table"] = k % 3 == 1, k % 4 == 2        # device engine: the dense SA, a 12-mer seed table (longer than -L 10)
    return c


def _odd_reads(c, contigs, reads, quals):
    """in place: the case's ragged lengths / Ns / contig-straddling reads (same treatment whatever the pairing)"""
    rng = np.random.default_rng(c.get("read_seed", 1))
    L = c["read_len"]
    joined = np.concatenate(contigs) if contigs else np.zeros(0, np.uint8)
    ends = np.cumsum([len(g) for g in contigs])[:-1]
    for i in range(len(reads)):
        r, q = reads[i].copy(), quals[i].copy()
        if c.get("straddle") and len(ends) and rng.random() < 0.08:
            e = int(rng.choice(ends)); a = max(0, e - int(rng.integers(1, L)))
            w = joined[a:a + L].copy()
            if len(w) == L:
                w = np.minimum(w, 4)
                r = (w if rng.random() < 0.5 else np.where(w[::-1] > 3, 4, 3 - np.minimum(w[::-1], 3))).astype(np.uint8)
        if c.get("n_rate", 0.0) > 0:
            r[rng.random(len(r)) < c["n_rate"]] = 4
        if c.get("ragged") and rng.random() < 0.5:
            n = int(rng.integers(0, len(r) + 1)) if rng.random() < 0.3 else int(rng.integers(max(1, len(r) // 2), len(r) + 1))
            if c["kw"].get("k") is not None or c["kw"].get("all_hits"):
                n = max(n, min(20, len(r)))      # (-a on a 2 bp read reports more alignments than align.py's per-read cap keeps)
            if c["paired"] and (i & 1) and n == 0 and not os.environ.get("BT2G_FUZZ_FILES"):
                n = 1          # an EMPTY mate 2 makes the reference treat the pair as an unpaired read (bt2_search.cpp:3326): the engines keep it a
                               # pair (DESIGN.md section 7); the file path (stream.TextAligner with its solo engine) follows the reference
            r, q = r[:n], q[:n]
        reads[i], quals[i] = np.ascontiguousarray(r, dtype=np.uint8), np.ascontiguousarray(q, dtype=np.uint8)


def _format_options(c, local):
    """what the record formatter has to know of the scoring options: the N ceiling (YF:Z:NS) and the shortest alignable read (YF:Z:SC)"""
    return {"sc": c["kw"]["sc"]} if "sc" in c["kw"] else {}


def _device_lines(c, base, batch, names, ref_names, fmt):
    """the case on the device engine (bt2g_xengine_*: the state machine in waves over the CUDA kernels, at the engine's own op-row
    width): align for -M, align_k + align.expand_entries for -k / -a.  -> (SAM records, (units, fallback units))"""
    from bowtie2_b200 import Bt2Gpu
    from bowtie2_b200.align import expand_entries, k_caps
    from bowtie2_b200.lib import XEngine, load_library, policy_params, sam_format
    lib = load_library()
    paired, kw = c["paired"], c["kw"]
    g = Bt2Gpu(0)
    try:
        g.load_index_files(base)
        if c.get("dense_sa"):
            g.build_dense_sa(0)
        if c.get("seed_table"):
            g.build_seed_table(12)
        prm = policy_params(c["preset"], local=c["local"], paired=paired, seed=c.get("run_seed", 0), **kw)
        units, max_len = batch.n // (2 if paired else 1), max(1, int(batch.lengths().max()))
        cap = k_caps(kw, paired)
        eng = XEngine(g, prm, units, max_len, max_per_unit=cap)
        try:
            if cap is None:
                res, ops, pairs, st = eng.align(batch, names)
                lines = sam_format(lib, batch, res, ops, ref_names, read_names=names, pairs=pairs, **fmt)
            else:
                res, ops, pairs, cnt, truncated, st = eng.align_k(batch, names)
                assert not truncated
                out = expand_entries(batch, names, res, ops, cnt, pairs)
                lines = sam_format(lib, out[0], out[2], out[3], ref_names, read_names=out[1], pairs=out[4] if paired else None, **fmt)
        finally:
            eng.close()
    finally:
        g.close()
    return lines.rstrip("\n").split("\n"), (units, st["fallback_units"])


def run_case(c, work, n_unpaired=300, n_pairs=200, device=False):
    """-> (records, differing, first difference or None, engine stats, description).  device: the device engine on the GPU
    (_device_lines) instead of the state machine's host build over the C oracle's table"""
    import conftest
    from bowtie2_b200 import synth
    from bowtie2_b200.lib import ReadBatch, load_library, policy_align, policy_params, sam_format
    lib = load_library()
    os.makedirs(work, exist_ok=True)
    contigs = synth.make_genome(n_contigs=c["n_contigs"], contig_len=c["contig_len"], seed=c["genome_seed"], repeat_frac=c["repeat_frac"],
                                repeat_len=c["repeat_len"], repeat_copies=c["repeat_copies"], n_gap=c["n_gap"])
    fa, base = os.path.join(work, "g.fa"), os.path.join(work, "g")
    synth.write_fasta(fa, contigs)
    large = c.get("large", False)
    for f in os.listdir(work):                                     # (a stale index of the other kind would be opened first)
        if f.startswith("g.") and (f.endswith(".bt2") or f.endswith(".bt2l")):
            os.remove(os.path.join(work, f))
    conftest._build_index("bowtie2-build-l" if large else "bowtie2-build-s", fa, base)
    ref_names = [f"chr{k + 1}" for k in range(len(contigs))]
    local, paired, L = c["local"], c["paired"], c["read_len"]
    if paired:
        reads, quals, _ = synth.make_pairs(contigs, n_pairs, L, seed=c["genome_seed"] + 1, sub_rate=c["sub_rate"], indel_rate=c["indel_rate"],
                                           ins_mean=c["ins_mean"], hard_frac=c["hard_frac"])
        _odd_reads(c, contigs, reads, quals)
        f1, f2 = os.path.join(work, "r1.fq"), os.path.join(work, "r2.fq")
        synth.write_fastq(f1, reads[0::2], quals[0::2], prefix="p"); synth.write_fastq(f2, reads[1::2], quals[1::2], prefix="p")
        names, inp = [f"p{i // 2}" for i in range(2 * n_pairs)], ["-1", f1, "-2", f2]
    else:
        reads, quals, _ = synth.make_reads(contigs, n_unpaired, L, seed=c["genome_seed"] + 1, sub_rate=c["sub_rate"], indel_rate=c["indel_rate"], random_frac=0.03)
        _odd_reads(c, contigs, reads, quals)
        f1 = os.path.join(work, "r.fq")
        synth.write_fastq(f1, reads, quals)
        names, inp = [f"r{i}" for i in range(n_unpaired)], ["-U", f1]
    pflag = "--" + c["preset"] + ("-local" if local else "")
    sam = os.path.join(work, "ref.sam")
    subprocess.check_call([REF[:-1] + "l" if large else REF, pflag] + (["--local"] if local else []) + c["flags"] + ["--seed", str(c.get("run_seed", 0)), "-p", "1", "--reorder", "-x", base] + inp + ["-S", sam],
                          stdout=subprocess.DEVNULL, stderr=open(os.path.join(work, "ref.err"), "w"))
    golden = [l.rstrip("\n") for l in open(sam) if not l.startswith("@")]
    from oracle_lib import Oracle, oracle_policy_table
    fmt = dict(local=local, no_discordant=(c["kw"].get("discord") is False), **_format_options(c, local))
    batch = ReadBatch.from_list(reads, quals)
    if device:
        lines, st = _device_lines(c, base, batch, names, ref_names, fmt)
    elif c["kw"].get("k") is not None or c["kw"].get("all_hits"):
        # every reported alignment: align.py's own expansion of bt2g_policy_align_k / bt2g_policy_align_pairs_k over the C oracle's table
        from bowtie2_b200.align import _exact_batch

        class _OracleDevice:
            _lib = lib

            def __init__(self):
                self.O, self.sc = Oracle(base), c["kw"].get("sc")

            def set_scoring_policy(self, sc, loc):
                self.sc = sc if "sc" in c["kw"] else None

            def policy_backend_table(self):
                return oracle_policy_table(self.O, local, 8 if large else 4, self.sc)
        out = _exact_batch(_OracleDevice(), batch, names, paired, c["preset"], local, c.get("run_seed", 0), 1, dict(c["kw"]))
        st = (batch.n // (2 if paired else 1), 0, 0)
        if paired:
            batch_k, names_k, res, ops, pairs_e, _ = out
            lines = sam_format(lib, batch_k, res, ops, ref_names, read_names=names_k, pairs=pairs_e, **fmt).rstrip("\n").split("\n")
        else:
            batch_k, names_k, res, ops, _ = out
            lines = sam_format(lib, batch_k, res, ops, ref_names, read_names=names_k, **fmt).rstrip("\n").split("\n")
    else:
        be, keep = oracle_policy_table(Oracle(base), local, 8 if large else 4, c["kw"].get("sc"))        # the C oracle behind the entry-point table
        res, ops, pairs, st = policy_align(lib, be, policy_params(c["preset"], local=local, paired=paired, seed=c.get("run_seed", 0), **c["kw"]), batch, names,
                                           entry="bt2g_xengine_align_host", max_ops=4 * L + 64)   # (room for the op strings of cheap-gap scoring schemes)
        lines = sam_format(lib, batch, res, ops, ref_names, read_names=names, pairs=pairs, **fmt).rstrip("\n").split("\n")
        if os.environ.get("BT2G_FUZZ_FILES"):
            # the same case as FILES: stream.align_files_stream (FastqFiles -> bt2g_fastq_parse[_pairs]_mt -> engine -> bt2g_sam_format -> SAM file
            # + alignment summary) around the state machine; records and summary against the reference program's
            import io
            from bowtie2_b200.stream import align_files_stream

            class _Eng:
                def __init__(self, prm):
                    self.prm = prm

                def align(self, b, nm):
                    return policy_align(lib, be, self.prm, b, nm, entry="bt2g_xengine_align_host", max_ops=4 * L + 64)
            summ = io.StringIO()
            outp = os.path.join(work, "ours.sam")
            align_files_stream(base, outp, inp[1], inp[3] if paired else None, preset=c["preset"], local=local, engines=1, batch_units=int(c["genome_seed"] % 90) + 37,
                               max_read_len=4 * L, threads=2, seed=c.get("run_seed", 0), summary=summ, policy_options=dict(c["kw"]), gpu=object(),
                               make_engine=lambda prm, n, l: _Eng(prm))
            flines = [l.rstrip("\n") for l in open(outp) if not l.startswith("@")]

            def split(text):                       # every line but the documented "exactly 1" / ">1" split of the concordant pairs (DESIGN.md section 7)
                conc, rest = 0, []
                for l in text.split("\n"):
                    if "aligned concordantly exactly 1 time" in l or "aligned concordantly >1 times" in l:
                        conc += int(l.split()[0])
                    else:
                        rest.append(l)
                return conc, rest
            ref_summary = "".join(l for l in open(os.path.join(work, "ref.err")) if not l.startswith("Warning"))
            lines = flines                                     # (the file path is the one judged in this mode)
            if lines == golden and split(summ.getvalue()) != split(ref_summary):
                lines = lines + ["SUMMARY DIFFERS: " + repr(summ.getvalue())]
                golden = golden + ["SUMMARY DIFFERS: " + repr(ref_summary)]
        if os.environ.get("BT2G_FUZZ_BOTH"):
            # the coroutine engine (csrc/policy_engine.cpp, the fallback of the state machine and align_files' engine) on the same case
            res2, ops2, pairs2, _ = policy_align(lib, be, policy_params(c["preset"], local=local, paired=paired, seed=c.get("run_seed", 0), **c["kw"]), batch, names,
                                                 max_ops=4 * L + 64)
            lines2 = sam_format(lib, batch, res2, ops2, ref_names, read_names=names, pairs=pairs2, **fmt).rstrip("\n").split("\n")
            if lines2 != lines and len(lines2) == len(lines):          # (not comparable when the file path wrote solo reads: empty mate 2)
                lines = lines2 if lines == golden else lines           # (report whichever differs from the reference)
    run_case.last = (lines, golden)                                # (for a closer look at a failing case)
    diff = [i for i, (a, b) in enumerate(zip(lines, golden)) if a != b]
    nbad = len(diff) + abs(len(lines) - len(golden))
    first = (lines[diff[0]], golden[diff[0]]) if diff else None
    odd = "".join([" ragged" if c.get("ragged") else "", f" Ns={c['n_rate']}" if c.get("n_rate") else "", " straddle" if c.get("straddle") else ""])
    desc = f"{'.bt2l ' if large else ''}{pflag} --seed {c.get('run_seed', 0)} {' '.join(c['flags'])} paired={paired} L={L} sub={c['sub_rate']} indel={c['indel_rate']} contigs={len(contigs)}{odd}"
    return len(golden), nbad, first, st, desc


def main():
    args = [a for a in sys.argv[1:] if a != "--device"]
    device = "--device" in sys.argv[1:]
    seed, cases = int(args[0]) if len(args) > 0 else 1, int(args[1]) if len(args) > 1 else 20
    work = args[2] if len(args) > 2 else os.path.join(tempfile.gettempdir(), "bt2g_parity_fuzz")
    tot = bad = units = fallbacks = 0
    t0 = time.time()
    for k in range(cases):
        c = draw_case(seed, k)
        n, nb, first, st, desc = run_case(c, work, device=device)
        tot += n; bad += nb; units += st[0]; fallbacks += st[1]
        extra = "".join([" dense-SA" if c["dense_sa"] else "", " seed-table-12" if c["seed_table"] else ""]) if device else ""
        print(f"case {k}: {desc}{extra}: {n} records, {nb} differing; {st[0]} units, {st[1]} finished by the coroutine engine", flush=True)
        if first:
            print("  GOT ", first[0][:300]); print("  WANT", first[1][:300])
    print(json.dumps({"seed": seed, "cases": cases, "records": tot, "differing": bad, "units": units, "host_fallbacks": fallbacks,
                      "seconds": round(time.time() - t0, 1),
                      "engine": ("bt2g_xengine_align / _align_k (the device engine on the CUDA kernels)" if device else
                                 "bt2g_xengine_align_host (csrc/xengine.cuh on the CPU, oracle-backed table)"),
                      "reference": "oracle/_ref/bowtie2-align-s --seed 0 --reorder -p 1"}))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
