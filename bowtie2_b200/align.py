"""Reads in -> SAM out: the caller of the hot path for whole files (host plumbing around include/bt2g.h).

FASTQ text (optionally gzip) is parsed in batches (bt2g_fastq_parse), each batch goes through the pipeline
(bt2g_pipeline_run_host / _run_paired_host: copies and kernels overlapped inside), the records are formatted by
bt2g_sam_format on host threads and written behind the header (bt2g_sam_header); the alignment summary
(bt2g_align_summary) is what the reference prints on stderr.  This is the part of multiseedSearchWorker
(bt2_search.cpp:3101-4100) that surrounds the search: read a batch, align, report, in input order.
Nothing here computes alignments; without a GPU `Bt2Gpu` raises before any file is opened for writing."""
import gzip
import os
import io
import sys

import numpy as np

from .lib import (ALIGN_COUNTS, Bt2Gpu, IndexFile, Pipeline, ReadBatch, align_counts_add, align_summary, fastq_parse,
                  load_library, sam_format, sam_header)


class FastqStream:
    """Batches of whole FASTQ records from a file (plain or .gz)."""

    def __init__(self, path: str, chunk_bytes: int = 32 << 20, name_stride: int = 256, threads: int = 1):
        self._f = gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")
        self._buf = b""
        self._eof = False
        self._chunk = chunk_bytes
        self._stride = name_stride
        self._threads = threads
        self._lib = load_library()

    def next_batch(self, max_reads: int):
        """-> (ReadBatch, names) with up to max_reads records; an empty batch at the end of the file."""
        while not self._eof and self._buf.count(b"\n") < 4 * max_reads + 4:
            more = self._f.read(self._chunk)
            if not more:
                self._eof = True
                break
            self._buf += more
        if self._eof and self._buf and not self._buf.endswith(b"\n"):
            self._buf += b"\n"                                   # last record without a final newline
        if not self._buf.strip():
            from .lib import NameTable
            return ReadBatch(np.zeros(0, np.uint8), np.zeros(1, np.uint64), np.zeros(0, np.uint8)), NameTable(np.zeros((0, self._stride), np.uint8))
        batch, names, used = fastq_parse(self._lib, self._buf, max_reads=max_reads, name_stride=self._stride, threads=self._threads)
        if batch.n == 0 and self._eof:
            raise RuntimeError("truncated FASTQ record at the end of the input")
        self._buf = self._buf[used:]
        return batch, names

    def close(self):
        self._f.close()


def interleave(b1: ReadBatch, b2: ReadBatch) -> ReadBatch:
    """mate 1 of pair i -> read 2i, mate 2 -> read 2i+1 (the layout bt2g_pipeline_run_paired_* takes)"""
    if b1.n != b2.n:
        raise ValueError(f"mate files differ in length within a batch ({b1.n} vs {b2.n} records)")
    n = b1.n
    l1, l2 = b1.lengths(), b2.lengths()
    lens = np.empty(2 * n, dtype=np.uint64)
    lens[0::2], lens[1::2] = l1, l2
    off = np.zeros(2 * n + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    total = int(off[-1])
    seq = np.empty(total, dtype=np.uint8)
    qual = np.empty(total, dtype=np.uint8)
    for b, l, start in ((b1, l1, off[0:2 * n:2]), (b2, l2, off[1:2 * n:2])):
        src0 = b.off[:-1].astype(np.int64)
        dst = np.repeat(start.astype(np.int64) - src0, l) + np.arange(int(b.off[-1]), dtype=np.int64)
        seq[dst] = b.seq[:int(b.off[-1])]
        qual[dst] = b.qual[:int(b.off[-1])]
    return ReadBatch(seq, off, qual)


def interleave_names(n1, n2):
    """names of mate 1 / mate 2 interleaved, as a NameTable (no per-name Python work)"""
    from .lib import NameTable
    rows = np.empty((2 * len(n1), n1.rows.shape[1]), dtype=np.uint8)
    rows[0::2], rows[1::2] = n1.rows, n2.rows
    return NameTable(rows)


ALL_HITS_CAP = 1024            # records per read kept for -a in exact mode (a warning is printed when a read had more)
ALL_HITS_CAP_PAIRS = 256      # report entries per pair kept for paired -a


def k_caps(options, paired):
    """entries kept per read (unpaired) or pair (paired) for -k N / -a: N, or 2N + 2 entries per pair (the primaries, then up to N - 1
    further records of each mate beside the other mate's primary, and an unaligned mate's own record); None outside -k / -a"""
    if not options or (options.get("k") is None and not options.get("all_hits")):
        return None
    if options.get("k") is not None:
        return int(options["k"]) * 2 + 2 if paired else int(options["k"])
    return ALL_HITS_CAP_PAIRS if paired else ALL_HITS_CAP


def gather_reads(batch, idx):
    """reads `idx` of a batch (repeats allowed), in that order, as a new ReadBatch"""
    o = batch.off.astype(np.int64)
    idx = np.asarray(idx, dtype=np.int64)
    lens = o[idx + 1] - o[idx]
    off = np.zeros(len(idx) + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    src = np.repeat(o[idx] - off[:-1].astype(np.int64), lens) + np.arange(int(off[-1]), dtype=np.int64)
    return ReadBatch(batch.seq[src], off, None if batch.qual is None else batch.qual[src])


def expand_entries(batch, names, res_k, ops_k, cnt, pairs_k=None):
    """-k / -a entry arrays (bt2g_policy_align_k / _pairs_k, bt2g_xengine_align_k) -> one SAM record per row: each read (pair) repeated
    once per entry it reports, an unaligned read (a pair) once.  -> (ReadBatch, names, results, ops[, pair records]) for bt2g_sam_format;
    rows of a pair that are mate context only (found bit 9) are skipped by the formatter."""
    from .lib import NameTable
    per = np.maximum(np.asarray(cnt, dtype=np.int64), 1)
    unit = np.repeat(np.arange(len(per)), per)
    sub = np.arange(len(unit)) - np.repeat(np.cumsum(per) - per, per)
    ridx = unit if pairs_k is None else np.stack([2 * unit, 2 * unit + 1], axis=1).reshape(-1)
    if isinstance(names, NameTable):
        nm = NameTable(names.rows[ridx])
    else:
        lst = list(names)
        nm = [lst[i] for i in ridx]
    res_f = np.ascontiguousarray(res_k[unit, sub]).reshape(-1)
    ops_f = np.ascontiguousarray(ops_k[unit, sub]).reshape(len(ridx), -1)
    if pairs_k is None:
        return gather_reads(batch, ridx), nm, res_f, ops_f
    return gather_reads(batch, ridx), nm, res_f, ops_f, np.ascontiguousarray(pairs_k[unit, sub])


def _exact_batch(gpu, batch, names, paired, preset, local, seed, threads=1, options=None):
    """one batch through the exact search policy in waves (csrc/policy_engine.cpp: bt2g_policy_align) over the entry points of
    this library: every read's state machine advances together, each primitive runs as one batched call per wave"""
    from .lib import policy_align, policy_align_k, policy_backend_gpu, policy_params
    multi = bool(options and (options.get("k") is not None or options.get("all_hits")))
    if hasattr(gpu, "policy_backend_table"):                    # a stand-in device (tests): its own table
        be, keep = gpu.policy_backend_table()
    else:
        be, keep = policy_backend_gpu(gpu), None
    from . import policy
    sc = (options or {}).get("sc") or policy.Scoring.default(local)
    if hasattr(gpu, "set_scoring_policy"):
        gpu.set_scoring_policy(sc, local)                       # kernels score with the same scheme the policy reasons about
    else:
        gpu.set_scoring(local=local)
    try:
        prm = policy_params(preset, local=local, paired=paired, seed=seed, host_threads=threads, **(options or {}))
        if multi and paired:
            # paired -k N / -a (bt2g_policy_align_pairs_k): entries of two rows per pair (the primaries, then the further concordant pairs
            # or the mates' further alignments beside the opposite primary); rows that are mate context only are skipped by the formatter
            from .lib import policy_align_pairs_k
            cap = k_caps(options, True)
            res_k, ops_k, pairs_k, cnt, truncated, stats = policy_align_pairs_k(gpu._lib, be, prm, batch, names, cap)
            if truncated:
                sys.stderr.write(f"Warning: -a: pairs with more than {cap} report entries were cut to {cap}\n")
            batch_k, names_k, res_f, ops_f, pairs_f = expand_entries(batch, names, res_k, ops_k, cnt, pairs_k)
            return batch_k, names_k, res_f, ops_f, pairs_f, (np.ascontiguousarray(res_k[:, 0]).reshape(-1), np.ascontiguousarray(pairs_k[:, 0]))
        if multi:
            # unpaired -k N / -a (bt2g_policy_align_k): one record per reported alignment, the read repeated; -a is capped per read
            cap = k_caps(options, False)
            # the multi-hit arrays are dense (n x cap result rows + n x cap op rows): cut the batch so that they stay under ~4 GiB
            row_bytes = 56 + int(batch.lengths().max() if batch.n else 0) + 64
            max_n = max(1, (4 << 30) // (cap * row_bytes))
            if batch.n > max_n:
                outs = []
                o = batch.off.astype(np.int64)
                nm = list(names)
                for a in range(0, batch.n, max_n):
                    b = min(batch.n, a + max_n)
                    sub = ReadBatch(batch.seq[o[a]:o[b]], (batch.off[a:b + 1] - batch.off[a]).astype(np.uint64), batch.qual[o[a]:o[b]])
                    outs.append(_exact_batch(gpu, sub, nm[a:b], paired, preset, local, seed, threads, options))
                rb = ReadBatch.from_list([x for t in outs for x in [t[0].seq[int(t[0].off[i]):int(t[0].off[i + 1])] for i in range(t[0].n)]],
                                         [x for t in outs for x in [t[0].qual[int(t[0].off[i]):int(t[0].off[i + 1])] for i in range(t[0].n)]])
                return rb, [x for t in outs for x in t[1]], np.concatenate([t[2] for t in outs]), np.concatenate([t[3] for t in outs]), \
                    np.concatenate([t[4] for t in outs])
            res_k, ops_k, cnt, truncated, stats = policy_align_k(gpu._lib, be, prm, batch, names, cap)
            if truncated:
                sys.stderr.write(f"Warning: -a: reads with more than {cap} alignments were cut to {cap} records\n")
            batch_k, names_k, res_f, ops_f = expand_entries(batch, names, res_k, ops_k, cnt)
            return batch_k, names_k, res_f, ops_f, np.ascontiguousarray(res_k[:, 0])
        res, ops, pairs, stats = policy_align(gpu._lib, be, prm, batch, names)
    finally:
        pass
    return res, ops, pairs


def align_files(index_base: str, out_path: str, reads1: str, reads2: str = None, preset: str = "sensitive", local: bool = False,
                device: int = 0, batch_reads: int = 1 << 20, threads: int = 8, seed_table: int = 0, dense_sa: int = -1,
                offrate: int = -1, pg_cl: str = None, summary=sys.stderr, gpu: Bt2Gpu = None, exact: bool = False, seed: int = 0,
                policy_options: dict = None):
    """bowtie2 -x index_base (-U reads1 | -1 reads1 -2 reads2) -S out_path.  Returns the ALIGN_COUNTS record.

    exact=False: the batched speculative pipeline (fast; agrees with the reference on the confidently placed reads).
    exact=True: the reference's sequential search policy (policy_engine) with every primitive computed on the GPU through
    policy_backend_gpu.GpuBackend, read by read: records identical to the reference program's, at a small fraction of the
    pipeline's speed (intended for parity subsets until the policy runs as a device-side state machine).
    policy_options (exact mode): keyword arguments of lib.policy_params -- nofw, norc, mixed, discord, pe (a
    policy.PairedEndPolicy: -I / -X / --ff ...), mhits (-M), sc (a policy.Scoring: --mp / --rdg / --score-min ...)."""
    own = gpu is None
    gpu = gpu or Bt2Gpu(device)                                  # raises without a GPU: nothing below runs on the CPU
    lib = gpu._lib
    image = IndexFile(index_base, offrate)
    gpu.load_index_host(image)
    ref_names, ref_lens = image.ref_names, image.ref_lens
    image.close()
    if seed_table:
        gpu.build_seed_table(seed_table)
    if dense_sa >= 0:
        gpu.build_dense_sa(dense_sa)
    paired = reads2 is not None
    s1 = FastqStream(reads1, threads=max(1, threads // (2 if paired else 1)))
    s2 = FastqStream(reads2, threads=max(1, threads // 2)) if paired else None
    per_batch = batch_reads // 2 if paired else batch_reads
    counts = np.zeros(1, dtype=ALIGN_COUNTS)
    pipe, pipe_len = None, 0
    sam_names = [n.split()[0] if n.split() else n for n in ref_names]
    # --no-discordant / --no-mixed reach the record formatter and the summary too (pair_type 2 alone cannot tell a discordant pair)
    no_disc = bool(exact and policy_options and policy_options.get("discord") is False)
    no_mixed = bool(exact and policy_options and policy_options.get("mixed") is False)
    sc_opt = policy_options.get("sc") if exact and policy_options else None       # --ma / --score-min / --n-ceil decide the YF:Z: tags
    with open(out_path, "wb") as out:
        out.write(sam_header(lib, ref_names, ref_lens, pg_cl).encode())
        while True:
            b1, n1 = s1.next_batch(per_batch)
            if paired:
                b2, n2 = s2.next_batch(per_batch)
                if b1.n != b2.n:
                    raise RuntimeError("fewer reads in one mate file than in the other")
            if b1.n == 0:
                break
            batch = interleave(b1, b2) if paired else b1
            names = interleave_names(n1, n2) if paired else n1
            need = int(batch.lengths().max())
            if not exact and (pipe is None or need > pipe_len):
                if pipe is not None:
                    pipe.close()
                pipe_len = max(need, 32)
                pipe = Pipeline(gpu, preset, max_len=pipe_len, max_reads=max(batch_reads, 2), row_cap=16, range_max=16, local=local,
                                both_mates=paired)
                if paired:
                    pipe.enable_pairs()
            if exact and paired and policy_options and (policy_options.get("k") is not None or policy_options.get("all_hits")):
                batch_k, names_k, res, ops, pairs_e, (prim_res, prim_pairs) = _exact_batch(gpu, batch, names, paired, preset, local, seed, threads, policy_options)
                out.write(sam_format(lib, batch_k, res, ops, sam_names, read_names=names_k, pairs=pairs_e, threads=threads, local=local, as_bytes=True,
                                     no_discordant=no_disc, sc=sc_opt))
                align_counts_add(lib, counts, prim_res, prim_pairs, no_discordant=no_disc)
                continue
            if exact and not paired and policy_options and (policy_options.get("k") is not None or policy_options.get("all_hits")):
                batch_k, names_k, res, ops, primary = _exact_batch(gpu, batch, names, paired, preset, local, seed, threads, policy_options)
                out.write(sam_format(lib, batch_k, res, ops, sam_names, read_names=names_k, threads=threads, local=local, as_bytes=True, sc=sc_opt))
                align_counts_add(lib, counts, primary, None)
                continue
            if exact:
                res, ops, pairs = _exact_batch(gpu, batch, names, paired, preset, local, seed, threads, policy_options)
            elif paired:
                res, ops, pairs = pipe.run_paired_host(batch)
            else:
                (res, ops), pairs = pipe.run_host(batch), None
            out.write(sam_format(lib, batch, res, ops, sam_names, read_names=names, pairs=pairs, threads=threads, local=local, as_bytes=True,
                                 no_discordant=no_disc, sc=sc_opt))
            align_counts_add(lib, counts, res, pairs, no_discordant=no_disc)
    if pipe is not None:
        pipe.close()
    s1.close()
    if s2 is not None:
        s2.close()
    if summary is not None:
        summary.write(align_summary(lib, counts, discord=not no_disc, mixed=not no_mixed))
    if own:
        gpu.close()
    return counts


# ---- the reference's other read formats (pat.cpp: FastaPatternSource, RawPatternSource, TabbedPatternSource,
#      QseqPatternSource, VectorPatternSource, FastaContinuousPatternSource): host-side parsing into the same buffers.
#      Secondary formats: plain Python, whole text at a time.
_CODE = np.full(256, 4, dtype=np.uint8)
for _i, _c in enumerate("ACGT"):
    _CODE[ord(_c)] = _CODE[ord(_c.lower())] = _i


def _batch_from(seqs, quals):
    seq = [_CODE[np.frombuffer(s.replace(".", "N").encode(), dtype=np.uint8)] for s in seqs]
    q = [np.frombuffer((qq if qq is not None else "I" * len(s)).encode(), dtype=np.uint8) for s, qq in zip(seqs, quals)]
    return ReadBatch.from_list(seq, q)


def parse_reads(text: str, fmt: str, first_id: int = 0, fasta_cont=None):
    """-> (names, sequences, qualities or None, mate-2 sequences / qualities for paired tabbed records or None)
    fmt: fasta (-f), raw (-r), tab5 (--tab5), tab6 (--tab6), qseq (--qseq), cline (-c: comma-separated sequences),
    fastacont (-F k,i with fasta_cont = (k, i)).  Reads without a name get their 0-based ordinal, as in the reference."""
    names, seqs, quals = [], [], []
    mate2 = []
    if fmt == "fasta":
        name, cur = None, []
        # FastaPatternSource::parse never appends the last character of a record's buffer (pat.cpp:864-879): harmless when it
        # is the newline, but a file without a final newline loses the last base of its last read.  Reproduced.
        if text and not text.endswith(("\n", "\r")) and not text.rstrip("\n").split("\n")[-1].startswith(">"):
            text = text[:-1]
        for line in text.split("\n") + [">"]:
            line = line.rstrip("\r")
            if line.startswith(">"):
                if name is not None:
                    names.append(name or str(first_id + len(names)))
                    seqs.append("".join(cur)); quals.append(None)
                name, cur = line[1:], []
            elif name is not None:
                cur.append(line.strip())
    elif fmt == "raw":
        for line in text.split("\n"):
            line = line.strip()
            if line:
                names.append(str(first_id + len(names))); seqs.append(line); quals.append(None)
    elif fmt == "cline":
        for s in text.split(","):
            s = s.strip()
            if ":" in s:                                           # SEQ:QUAL
                s, q = s.split(":", 1)
            else:
                q = None
            names.append(str(first_id + len(names))); seqs.append(s); quals.append(q)
    elif fmt in ("tab5", "tab6"):
        for line in text.split("\n"):
            f = line.rstrip("\r").split("\t")
            if len(f) < 3:
                continue
            if len(f) == 3:
                names.append(f[0]); seqs.append(f[1]); quals.append(f[2]); mate2.append(None)
            elif len(f) == 5:
                names.append(f[0]); seqs.append(f[1]); quals.append(f[2]); mate2.append((f[0], f[3], f[4]))
            else:
                names.append(f[0]); seqs.append(f[1]); quals.append(f[2]); mate2.append((f[3], f[4], f[5]))
    elif fmt == "qseq":
        for line in text.split("\n"):
            f = line.rstrip("\r").split("\t")
            if len(f) < 11:
                continue
            names.append("_".join(f[0:7]) + "/" + f[7]); seqs.append(f[8]); quals.append(f[9])
    elif fmt == "fastacont":
        k, step = fasta_cont
        name, cur = None, []
        recs = []
        for line in text.split("\n") + [">"]:
            line = line.rstrip("\r")
            if line.startswith(">"):
                if name is not None:
                    recs.append((name.split()[0] if name.split() else name, "".join(cur)))
                name, cur = line[1:], []
            elif name is not None:
                cur.append(line.strip())
        for nm, s in recs:
            # FastaContinuousPatternSource: every window of k characters whose end offset is a multiple of the interval
            for end in range(k, len(s) + 1):
                off = end - k
                if off % step == 0:
                    names.append(f"{nm}_{off}"); seqs.append(s[off:end]); quals.append(None)
    else:
        raise ValueError(f"unknown read format {fmt}")
    return names, seqs, quals, (mate2 if any(m is not None for m in mate2) else None)
