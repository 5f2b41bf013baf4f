"""-k N / -a on the device engine's state machine (csrc/xengine.cuh), driven on the host by bt2g_xengine_align_host_k over the oracle's
entry-point tables: the report order kept by finishRead / finishPair and the entry writer x_report_entry (the function k_xe_report runs on
the GPU) give arrays byte-identical to the coroutine engine's bt2g_policy_align_k / _pairs_k, and SAM identical to the reference
program's."""
import subprocess

import numpy as np
import pytest

from bowtie2_b200 import synth
from bowtie2_b200.align import expand_entries
from bowtie2_b200.lib import ReadBatch, load_library, policy_align_k, policy_align_pairs_k, policy_params, sam_format, xengine_align_host_k
from fake_gpu import FakeGpu, backend_table
from oracle_lib import Oracle, have_reference, oracle_policy_table, ref_bin

pytestmark = pytest.mark.skipif(not have_reference(), reason="oracle/_ref not built")


@pytest.fixture(scope="module")
def genome_index(tmp_path_factory):
    """the repeat-rich synthetic genome of test_policy_engine_cpp.py (150-copy repeat families), indexed as .bt2 and .bt2l"""
    d = tmp_path_factory.mktemp("xk")
    genome = synth.make_genome(n_contigs=3, contig_len=60000, seed=11, repeat_frac=0.5, repeat_len=250, repeat_copies=150, n_gap=37)
    fa = str(d / "g.fa")
    synth.write_fasta(fa, genome)
    subprocess.check_call([ref_bin("bowtie2-build-s"), "--seed", "0", "--quiet", fa, str(d / "s")])
    subprocess.check_call([ref_bin("bowtie2-build-l"), "--seed", "0", "--quiet", fa, str(d / "l")])
    return genome, d


def _table(base, local, large, python_device):
    if python_device:                                        # the Python stand-in device (tests/fake_gpu.py)
        fake = FakeGpu(Oracle(base), 8 if large else 4)
        fake.set_scoring(local)
        be, keep = backend_table(fake)
        return be, (keep, fake)
    return oracle_policy_table(Oracle(base), local, 8 if large else 4)      # the plain-C restatement (oracle/bt2_oracle_table.c)


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert x.shape == y.shape and x.tobytes() == y.tobytes()
        else:
            assert x == y


# Units of these batches that the state machine hands to the coroutine engine (a sink list beyond XE_LIST = 64, a DP answer beyond its
# lists, a full arena).  The host twin is deterministic; observed: unpaired -k 3 8 of 200 (.bt2l: 7 of 150), -k 12 23 of 200,
# --local -k 5 21 of 150; paired -k 3 18 of 120, --local -k 5 14 of 80 (17.5 %); -a 37 of 120 unpaired, 30 of 80 paired (37.5 %).
MAX_FALLBACK_SHARE_K = 0.20
MAX_FALLBACK_SHARE_A = 0.40

CASES = [
    # (paired, local, large, reference args, policy kwargs, cap, reads, python stand-in device)
    (False, False, False, ["-k", "3"], dict(k=3), 3, 200, True),
    (False, False, False, ["-k", "12"], dict(k=12), 12, 200, False),
    (False, False, False, ["-a"], dict(all_hits=True), 400, 120, False),
    (True, False, False, ["-k", "3"], dict(k=3), 8, 120, True),
    (True, False, False, ["-a"], dict(all_hits=True), 256, 80, False),
    (False, True, False, ["--local", "-k", "5"], dict(k=5), 5, 150, False),
    (False, False, True, ["-k", "3"], dict(k=3), 3, 150, False),
    (True, True, False, ["--local", "-k", "5"], dict(k=5), 12, 80, False),
]


@pytest.mark.parametrize("paired,local,large,args,kw,cap,n,python_device", CASES,
                         ids=["U-k3-py", "U-k12", "U-a", "P-k3-py", "P-a", "U-local-k5", "U-bt2l-k3", "P-local-k5"])
def test_host_twin_equals_coroutine_engine_and_reference(genome_index, tmp_path, paired, local, large, args, kw, cap, n, python_device):
    genome, d = genome_index
    base = str(d / ("l" if large else "s"))
    if paired:
        reads, quals, _ = synth.make_pairs(genome, n, 100, seed=32, sub_rate=0.02, indel_rate=0.003, hard_frac=0.2, hard_period=12, ins_mean=300, ins_sd=90)
        names = [f"r{i // 2}" for i in range(2 * n)]
        f1, f2 = str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")
        synth.write_fastq(f1, reads[0::2], quals[0::2])
        synth.write_fastq(f2, reads[1::2], quals[1::2])
        inp = ["-1", f1, "-2", f2]
    else:
        reads, quals, _ = synth.make_reads(genome, n, 100, seed=79, sub_rate=0.02, indel_rate=0.003)
        names = [f"r{i}" for i in range(n)]
        fq = str(tmp_path / "r.fq")
        synth.write_fastq(fq, reads, quals)
        inp = ["-U", fq]
    preset = "--sensitive-local" if local else "--sensitive"
    out = subprocess.check_output([ref_bin("bowtie2-align-" + ("l" if large else "s")), preset, "--seed", "0", "-p", "1", "--reorder", "-x", base] + inp + args,
                                  stderr=subprocess.DEVNULL).decode()
    want = [l for l in out.split("\n") if l and not l.startswith("@")]
    ref_names = [l.split("\t")[1][3:] for l in out.split("\n") if l.startswith("@SQ")]
    lib = load_library()
    be, keep = _table(base, local, large, python_device)
    prm = policy_params("sensitive", local=local, paired=paired, k=kw.get("k"), all_hits=kw.get("all_hits", False))
    batch = ReadBatch.from_list(reads, quals)
    got = xengine_align_host_k(lib, be, prm, batch, names, cap)
    ref = (policy_align_pairs_k if paired else policy_align_k)(lib, be, prm, batch, names, cap)
    _same(got[:-1], ref[:-1])                                # arrays, entry counts, truncation flag (stats differ: units, fallbacks, requests)
    assert not got[-2]
    if paired:
        res, ops, pairs, cnt = got[:4]
        b, nm, r, o, p = expand_entries(batch, names, res, ops, cnt, pairs)
        lines = sam_format(lib, b, r, o, ref_names, read_names=nm, pairs=p, local=local).rstrip("\n").split("\n")
    else:
        res, ops, cnt = got[:3]
        b, nm, r, o = expand_entries(batch, names, res, ops, cnt)
        lines = sam_format(lib, b, r, o, ref_names, read_names=nm, local=local).rstrip("\n").split("\n")
    diff = [(a, w) for a, w in zip(lines, want) if a != w]
    assert len(lines) == len(want) and not diff, (len(lines), len(want), diff[:1])
    assert sum(int(l.split("\t")[1]) & 256 != 0 for l in want) > 10     # secondaries were reported
    # the units that fall back are answered by the coroutine engine itself: the equality above pins the state machine only on the others
    units, fallbacks, _ = got[-1]
    assert units == n and fallbacks <= (MAX_FALLBACK_SHARE_A if kw.get("all_hits") else MAX_FALLBACK_SHARE_K) * units, (fallbacks, units)


@pytest.mark.parametrize("paired", [False, True])
def test_cap_below_the_alignment_count_truncates_like_the_coroutine_engine(genome_index, paired):
    genome, d = genome_index
    base = str(d / "s")
    if paired:
        reads, quals, _ = synth.make_pairs(genome, 80, 100, seed=32, sub_rate=0.02, indel_rate=0.003, ins_mean=300, ins_sd=90)
        names = [f"r{i // 2}" for i in range(len(reads))]
    else:
        reads, quals, _ = synth.make_reads(genome, 150, 100, seed=79, sub_rate=0.02, indel_rate=0.003)
        names = [f"r{i}" for i in range(len(reads))]
    lib = load_library()
    be, keep = _table(base, False, False, False)
    prm = policy_params("sensitive", paired=paired, k=12)
    batch = ReadBatch.from_list(reads, quals)
    got = xengine_align_host_k(lib, be, prm, batch, names, 2)
    ref = (policy_align_pairs_k if paired else policy_align_k)(lib, be, prm, batch, names, 2)
    _same(got[:-1], ref[:-1])
    cnt = got[3] if paired else got[2]
    assert got[-2] and int(cnt.max()) == 2


def test_parity_fuzz_k_cases_through_the_host_twin(tmp_path, monkeypatch):
    """the -k / -a cases of the parity fuzz (seed 101: cases 11, 44, 55) with align.py's -k step answered by bt2g_xengine_align_host_k
    instead of the coroutine engine: every record identical to the reference program's"""
    import parity_fuzz
    from bowtie2_b200 import align as align_mod
    from bowtie2_b200.align import k_caps

    def host_k_batch(gpu, batch, names, paired, preset, local, seed, threads=1, options=None):
        be, keep = gpu.policy_backend_table()
        prm = policy_params(preset, local=local, paired=paired, seed=seed, host_threads=threads, **options)
        cap = k_caps(options, paired)
        out = xengine_align_host_k(gpu._lib, be, prm, batch, names, cap)
        assert not out[-2]
        host_k_batch.units += out[-1][0]
        host_k_batch.fallbacks += out[-1][1]
        if paired:
            res, ops, pairs, cnt = out[:4]
            return (*expand_entries(batch, names, res, ops, cnt, pairs), None)
        res, ops, cnt = out[:3]
        return (*expand_entries(batch, names, res, ops, cnt), None)
    host_k_batch.units = host_k_batch.fallbacks = 0
    monkeypatch.setattr(align_mod, "_exact_batch", host_k_batch)
    for k in (11, 44, 55):
        c = parity_fuzz.draw_case(101, k)
        assert c["kw"].get("k") is not None or c["kw"].get("all_hits"), c["flags"]
        n, nbad, first, st, desc = parity_fuzz.run_case(c, str(tmp_path / f"c{k}"))
        assert nbad == 0, (k, desc, first)
    assert host_k_batch.units > 0 and host_k_batch.fallbacks < host_k_batch.units


class _HostKEngine:
    """a -k / -a engine for the stream loop without a GPU: align_k answered by bt2g_xengine_align_host_k over the oracle's table"""

    def __init__(self, be, prm, lock, max_units, max_per_unit):
        self.be, self.prm, self.lock, self.max_units, self.max_per_unit = be, prm, lock, max_units, max_per_unit

    def align_k(self, batch, names):
        with self.lock:                                      # (one oracle table, several aligner threads)
            out = xengine_align_host_k(load_library(), self.be, self.prm, batch, list(names), self.max_per_unit)
        if self.prm.paired:
            res, ops, pairs, cnt, truncated, st = out
        else:
            (res, ops, cnt, truncated, st), pairs = out, None
        return res, ops, pairs, cnt, truncated, {"fallback_units": st[1]}


def _summary_split(text):
    """the alignment summary, but for the documented "exactly 1" / ">1" split of the concordant pairs (DESIGN.md section 7)"""
    conc, rest = 0, []
    for l in text.split("\n"):
        if "aligned concordantly exactly 1 time" in l or "aligned concordantly >1 times" in l:
            conc += int(l.split()[0])
        elif l and not l.startswith("Warning"):
            rest.append(l)
    return conc, rest


@pytest.mark.parametrize("paired,empty_mates", [(False, ()), (True, (0, 17, 18, 36, 63, 99))],
                         ids=["unpaired-k3", "paired-k3-empty-mate-2"])
def test_align_files_stream_k3_equals_the_reference(genome_index, tmp_path, paired, empty_mates):
    """align_files_stream with -k 3 over two engines and uneven batches (the stream loop, entry expansion and alignment counts around
    the state machine): SAM records and alignment summary equal the reference program's.  Pairs whose mate 2 is empty are unpaired
    reads for the reference; they go through the unpaired -k solo engine and leave their records in place."""
    import io
    import threading
    from bowtie2_b200.stream import align_files_stream
    genome, d = genome_index
    base = str(d / "s")
    if paired:
        reads, quals, _ = synth.make_pairs(genome, 100, 100, seed=32, sub_rate=0.02, indel_rate=0.003, hard_frac=0.2, hard_period=12, ins_mean=300, ins_sd=90)
        for i in empty_mates:
            reads[2 * i + 1], quals[2 * i + 1] = reads[2 * i + 1][:0], quals[2 * i + 1][:0]
        f1, f2 = str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")
        synth.write_fastq(f1, reads[0::2], quals[0::2])
        synth.write_fastq(f2, reads[1::2], quals[1::2])
        inp = ["-1", f1, "-2", f2]
    else:
        reads, quals, _ = synth.make_reads(genome, 150, 100, seed=79, sub_rate=0.02, indel_rate=0.003)
        f1, f2 = str(tmp_path / "r.fq"), None
        synth.write_fastq(f1, reads, quals)
        inp = ["-U", f1]
    ref = subprocess.run([ref_bin("bowtie2-align-s"), "--sensitive", "--seed", "0", "-p", "1", "--reorder", "-x", base] + inp + ["-k", "3"],
                         capture_output=True, check=True)
    want = [l for l in ref.stdout.decode().split("\n") if l and not l.startswith("@")]
    be, keep = _table(base, False, False, False)
    lock = threading.Lock()
    made = []

    def make_engine(prm, max_units, max_len, max_per_unit=None):
        assert max_per_unit is not None                      # -k: every engine, the solo engine included, reports entries
        made.append((bool(prm.paired), max_per_unit))
        return _HostKEngine(be, prm, lock, max_units, max_per_unit)
    out, summ = str(tmp_path / "ours.sam"), io.StringIO()
    align_files_stream(base, out, f1, f2, engines=2, batch_units=37, max_read_len=128, threads=3, summary=summ, policy_options={"k": 3},
                       gpu=object(), make_engine=make_engine)
    got = [l.rstrip("\n") for l in open(out) if not l.startswith("@")]
    diff = [(a, w) for a, w in zip(got, want) if a != w]
    assert len(got) == len(want) and not diff, (len(got), len(want), diff[:1])
    assert _summary_split(summ.getvalue()) == _summary_split(ref.stderr.decode())
    assert sum(int(l.split("\t")[1]) & 256 != 0 for l in want) > 10
    if empty_mates:
        assert (False, 3) in made and sum("YT:Z:UU" in l for l in got) >= len(empty_mates)     # the unpaired -k solo engine wrote them
