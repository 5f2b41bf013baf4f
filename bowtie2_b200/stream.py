"""FASTQ text in -> SAM text out around the device engine, with the host stages overlapped on threads:

    parse (bt2g_fastq_parse_mt / bt2g_fastq_parse_pairs_mt: the two mate files straight into one interleaved batch)
      ||  align (bt2g_xengine_align, one host thread per engine)  ||  format (bt2g_sam_format)

Every stage is one call into libbt2g.so per batch (ctypes releases the GIL), so the threads run concurrently; batches leave in
input order.  This is the batch loop of multiseedSearchWorker (bt2_search.cpp:3253-4254) with its reader
(PatternSourcePerThread, pat.cpp) and its sink (AlnSinkSam, aln_sink.cpp:1889) -- host plumbing: nothing here computes
alignments."""
import inspect
import queue
import sys
import threading

import numpy as np

from .lib import HostBuffers, NameTable, ReadBatch, XEngine, fastq_parse, fastq_parse_pairs, load_library, sam_format


def interleave_uniform(b1: ReadBatch, b2: ReadBatch, n1: NameTable, n2: NameTable):
    """mate 1 of pair i -> read 2i, mate 2 -> read 2i + 1; fast path for batches whose reads all have one length per file"""
    n = b1.n
    if n != b2.n:
        raise ValueError(f"mate files differ in length within a batch ({b1.n} vs {b2.n} records)")
    l1, l2 = b1.lengths(), b2.lengths()
    if n and (l1 == l1[0]).all() and (l2 == l2[0]).all() and l1[0] == l2[0]:
        L = int(l1[0])
        seq = np.empty((n, 2, L), dtype=np.uint8)
        qual = np.empty((n, 2, L), dtype=np.uint8)
        seq[:, 0], seq[:, 1] = b1.seq[:n * L].reshape(n, L), b2.seq[:n * L].reshape(n, L)
        qual[:, 0], qual[:, 1] = b1.qual[:n * L].reshape(n, L), b2.qual[:n * L].reshape(n, L)
        batch = ReadBatch(seq.reshape(-1), np.arange(0, (2 * n + 1) * L, L, dtype=np.uint64), qual.reshape(-1))
    else:
        from .align import interleave
        batch = interleave(b1, b2)
    rows = np.empty((2 * n, n1.rows.shape[1]), dtype=np.uint8)
    rows[0::2], rows[1::2] = n1.rows, n2.rows
    return batch, NameTable(rows)


class TextAligner:
    """engines: list of XEngine (all created with the same parameters); ref_names: @SQ names in index order.
    Every batch in flight owns one set of reused host buffers (lib.HostBuffers: parsed reads, names, results), and the SAM text
    of a batch is handed to the sink as a memoryview of one reused output buffer: the sink must consume it (write it) before it
    returns.  No per-batch allocation is left on the steady-state path."""

    def __init__(self, engines, ref_names, paired, local=False, parse_threads=4, format_threads=8, name_stride=32, depth=2, no_discordant=False, sc=None, make_solo_engine=None,
                 policy_options=None):
        """policy_options: the run's options; with {"k": N} or {"all_hits": True} the engines (and the solo engine) are -k / -a engines (XEngine
        with max_per_unit: align_k) and every reported alignment is written, the read or pair repeated per entry (align.expand_entries).
        make_solo_engine: () -> an UNPAIRED engine (same preset and options), created on first use.  A pair whose mate 2 is empty is an
        unpaired read for the reference (`paired = !read_b().empty()`, bt2_search.cpp:3326: mate 1 goes through the unpaired policy and
        leaves ONE record, YT:Z:UU, counted with the unpaired reads); with the factory those pairs are aligned and written that way,
        without it they stay pairs (two records, mate 2 unaligned with YF:Z:LN)."""
        self.engines, self.ref_names, self.paired, self.local = list(engines), list(ref_names), paired, local
        self.make_solo_engine, self._solo, self._solo_lock = make_solo_engine, None, threading.Lock()
        self.parse_threads, self.format_threads, self.name_stride, self.depth = parse_threads, format_threads, name_stride, depth
        self.no_discordant, self.sc = no_discordant, sc          # the run's --no-discordant / scoring scheme, for the record formatter
        self.multi = bool(policy_options and (policy_options.get("k") is not None or policy_options.get("all_hits")))
        self.lib = load_library()
        self._slots = [HostBuffers() for _ in range(depth + len(self.engines) + 1)]
        # (engine stand-ins of the CPU tests may not take reusable result buffers)
        self._reuse = [(not self.multi and "out" in inspect.signature(e.align).parameters) for e in self.engines]
        self._out = HostBuffers()

    def _parse(self, item, slot):
        t1, t2 = item
        if not self.paired:
            b1, n1, used1 = fastq_parse(self.lib, t1, name_stride=self.name_stride, threads=self.parse_threads, out=slot)
            if used1 != len(t1):
                raise ValueError(f"FASTQ text of a batch ends inside a record (byte {used1} of {len(t1)})")
            return b1, n1
        batch, names, used1, used2 = fastq_parse_pairs(self.lib, t1, t2, name_stride=self.name_stride, threads=self.parse_threads, out=slot)
        if used1 != len(t1) or used2 != len(t2):
            raise ValueError(f"mate files differ in length within a batch ({batch.n // 2} whole pairs; {len(t1) - used1} and {len(t2) - used2} bytes left over)")
        return batch, names

    def _align_solos(self, batch, names):
        """the pairs of a batch whose mate 2 is empty, their mate 1 aligned as unpaired reads: None, or (pair indexes, ReadBatch, names,
        results, ops)"""
        ln = batch.lengths()
        idx = np.nonzero(ln[1::2] == 0)[0]
        if len(idx) == 0:
            return None
        o = batch.off.astype(np.int64)
        sb = ReadBatch.from_list([batch.seq[o[2 * i]:o[2 * i + 1]] for i in idx], [batch.qual[o[2 * i]:o[2 * i + 1]] for i in idx])
        sn = NameTable(np.ascontiguousarray(names.rows[2 * idx])) if isinstance(names, NameTable) else [names[2 * int(i)] for i in idx]
        with self._solo_lock:                                    # (one unpaired engine, shared by the aligner threads: such pairs are rare)
            if self._solo is None:
                self._solo = self.make_solo_engine()
            cap = int(getattr(self._solo, "max_units", 1 << 30))
            parts = []
            for a in range(0, sb.n, cap):
                b = min(sb.n, a + cap)
                so = sb.off.astype(np.int64)
                part = ReadBatch(sb.seq[so[a]:so[b]], (sb.off[a:b + 1] - sb.off[a]).astype(np.uint64), sb.qual[so[a]:so[b]])
                r, op, _, _ = self._solo.align(part, sn[a:b])
                parts.append((np.array(r, copy=True), np.array(op, copy=True)))
        width = max(p[1].shape[1] for p in parts)
        ops = np.zeros((sb.n, width), dtype=np.uint8)
        at = 0
        for r, op in parts:
            ops[at:at + len(r), :op.shape[1]] = op
            at += len(r)
        return idx, sb, sn, np.concatenate([p[0] for p in parts]), ops

    @staticmethod
    def _warn_truncated(eng, paired):
        cap = eng.max_per_unit
        if paired:
            sys.stderr.write(f"Warning: -a: pairs with more than {cap} report entries were cut to {cap}\n")
        else:
            sys.stderr.write(f"Warning: -a: reads with more than {cap} alignments were cut to {cap} records\n")

    def _k_segments(self, eng, batch, names):
        """-k / -a: the batch through align_k, expanded to one record per row, as the formatter's segments (ReadBatch, names, res, ops,
        pairs or None, primary results and pair records for the alignment counts: entry 0 of every unit), in input order"""
        from .align import expand_entries
        res, ops, pairs, cnt, truncated, _ = eng.align_k(batch, names)
        if truncated:
            self._warn_truncated(eng, self.paired)
        if not self.paired:
            return [(*expand_entries(batch, names, res, ops, cnt), None, np.ascontiguousarray(res[:, 0]), None)]
        solo = None
        if self.make_solo_engine is not None:
            idx = np.nonzero(batch.lengths()[1::2] == 0)[0]
            if len(idx):
                solo = (idx, *self._align_solos_k(batch, names, idx))
        o = batch.off.astype(np.int64)

        def pairs_run(a, b):                                     # pairs [a, b)
            sb = ReadBatch(batch.seq[o[2 * a]:o[2 * b]], (batch.off[2 * a:2 * b + 1] - batch.off[2 * a]).astype(np.uint64), batch.qual[o[2 * a]:o[2 * b]])
            return (*expand_entries(sb, names[2 * a:2 * b], res[a:b], ops[a:b], cnt[a:b], pairs[a:b]),
                    np.ascontiguousarray(res[a:b, 0]).reshape(-1), np.ascontiguousarray(pairs[a:b, 0]))
        if solo is None:
            return [pairs_run(0, batch.n // 2)]
        idx, sb, sn, sres, sops, scnt = solo
        so = sb.off.astype(np.int64)
        segs, prev = [], 0
        for j, p in enumerate(int(x) for x in idx):
            if p > prev:
                segs.append(pairs_run(prev, p))
            one = ReadBatch(sb.seq[so[j]:so[j + 1]], (sb.off[j:j + 2] - sb.off[j]).astype(np.uint64), sb.qual[so[j]:so[j + 1]])
            segs.append((*expand_entries(one, sn[j:j + 1], sres[j:j + 1], sops[j:j + 1], scnt[j:j + 1]), None, np.ascontiguousarray(sres[j:j + 1, 0]), None))
            prev = p + 1
        if prev < batch.n // 2:
            segs.append(pairs_run(prev, batch.n // 2))
        return segs

    def _align_solos_k(self, batch, names, idx):
        """-k / -a: mate 1 of the pairs `idx` (empty mate 2) through the unpaired solo engine: (ReadBatch, names, res, ops, n_entries)"""
        o = batch.off.astype(np.int64)
        sb = ReadBatch.from_list([batch.seq[o[2 * i]:o[2 * i + 1]] for i in idx], [batch.qual[o[2 * i]:o[2 * i + 1]] for i in idx])
        sn = NameTable(np.ascontiguousarray(names.rows[2 * idx])) if isinstance(names, NameTable) else [names[2 * int(i)] for i in idx]
        with self._solo_lock:
            if self._solo is None:
                self._solo = self.make_solo_engine()
            cap = int(getattr(self._solo, "max_units", 1 << 30))
            parts = []
            for a in range(0, sb.n, cap):
                b = min(sb.n, a + cap)
                so = sb.off.astype(np.int64)
                part = ReadBatch(sb.seq[so[a]:so[b]], (sb.off[a:b + 1] - sb.off[a]).astype(np.uint64), sb.qual[so[a]:so[b]])
                r, op, _, cnt, truncated, _ = self._solo.align_k(part, sn[a:b])
                if truncated:
                    self._warn_truncated(self._solo, False)
                parts.append((r, op, cnt))
        return sb, sn, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), np.concatenate([p[2] for p in parts])

    @staticmethod
    def _segments(batch, names, res, ops, pairs, solo):
        """the batch as runs of ordinary pairs with the solo reads between them, in input order: (ReadBatch, names, res, ops, pairs or None)"""
        idx, sb, sn, sres, sops = solo
        o = batch.off.astype(np.int64)

        def pairs_run(a, b):                                     # pairs [a, b)
            return (ReadBatch(batch.seq[o[2 * a]:o[2 * b]], (batch.off[2 * a:2 * b + 1] - batch.off[2 * a]).astype(np.uint64), batch.qual[o[2 * a]:o[2 * b]]),
                    names[2 * a:2 * b], res[2 * a:2 * b], ops[2 * a:2 * b], pairs[a:b])
        so = sb.off.astype(np.int64)
        prev = 0
        for j, p in enumerate(int(x) for x in idx):
            if p > prev:
                yield pairs_run(prev, p)
            yield (ReadBatch(sb.seq[so[j]:so[j + 1]], (sb.off[j:j + 2] - sb.off[j]).astype(np.uint64), sb.qual[so[j]:so[j + 1]]), sn[j:j + 1],
                   sres[j:j + 1], sops[j:j + 1], None)
            prev = p + 1
        if prev < batch.n // 2:
            yield pairs_run(prev, batch.n // 2)

    def run(self, items, sink, on_batch=None):
        """items: iterable of (mate-1 FASTQ text, mate-2 FASTQ text or None), each at most one engine batch -- or a FastqFiles object
        (whole files, cut into batches here); sink(view) is called once per batch (more often for a batch with solo reads, see
        make_solo_engine), in input order, with the SAM text as a memoryview that is valid until the sink returns; on_batch(res, pairs),
        if given, sees the result arrays behind every sink call first (the alignment summary's counts).  Returns the number of reads written."""
        q_free, q_parsed, q_done = queue.Queue(), queue.Queue(), queue.Queue()
        for slot in self._slots:
            q_free.put(slot)
        errs, total = [], [0]
        END = object()

        def parser():
            try:
                if isinstance(items, FastqFiles):
                    k = 0
                    while True:
                        slot = q_free.get()                      # (back-pressure: at most len(slots) batches in flight)
                        if errs:
                            break
                        got = items.next_batch(self.lib, slot, self.name_stride, self.parse_threads)
                        if got is None:
                            q_free.put(slot)
                            break
                        q_parsed.put((k, slot, *got))
                        k += 1
                else:
                    for k, item in enumerate(items):
                        slot = q_free.get()
                        if errs:
                            break
                        q_parsed.put((k, slot, *self._parse(item, slot)))
            except Exception as e:
                errs.append(e)
            for _ in self.engines:
                q_parsed.put(END)

        def aligner(eng, reuse):
            try:
                while True:
                    w = q_parsed.get()
                    if w is END:
                        break
                    k, slot, batch, names = w
                    if self.multi:                               # -k / -a: segments of expanded records, ready for the formatter
                        q_done.put((k, slot, batch, names, None, None, None, self._k_segments(eng, batch, names)))
                        continue
                    res, ops, pairs, _ = eng.align(batch, names, out=slot) if reuse else eng.align(batch, names)
                    solo = self._align_solos(batch, names) if self.paired and self.make_solo_engine is not None else None
                    q_done.put((k, slot, batch, names, res, ops, pairs, solo))
            except Exception as e:
                errs.append(e)
                q_free.put(HostBuffers())                        # never leave the parser waiting
            q_done.put(END)

        def formatter():
            try:
                pending, nxt, ended = {}, 0, 0
                while ended < len(self.engines):
                    w = q_done.get()
                    if w is END:
                        ended += 1
                        continue
                    pending[w[0]] = w[1:]
                    while nxt in pending:
                        slot, batch, names, res, ops, pairs, solo = pending.pop(nxt)
                        if res is None:                          # -k / -a: the aligner's segments (counted by their primaries)
                            segs = solo
                        else:
                            segs = [(batch, names, res, ops, pairs)] if solo is None else self._segments(batch, names, res, ops, pairs, solo)
                            segs = [(*sg, sg[2], sg[4]) for sg in segs]
                        for b_, n_, r_, o_, p_, cr_, cp_ in segs:
                            txt = sam_format(self.lib, b_, r_, o_, self.ref_names, read_names=n_, pairs=p_, threads=self.format_threads,
                                             local=self.local, as_bytes="view", out=self._out, no_discordant=self.no_discordant, sc=self.sc)
                            if on_batch is not None:
                                on_batch(cr_, cp_)
                            sink(txt)
                        total[0] += batch.n
                        nxt += 1
                        del batch, names, res, ops, pairs, solo
                        q_free.put(slot)
            except Exception as e:
                errs.append(e)
                for _ in range(len(self._slots)):
                    q_free.put(HostBuffers())

        th = [threading.Thread(target=parser)] + [threading.Thread(target=aligner, args=(e, r)) for e, r in zip(self.engines, self._reuse)] + [threading.Thread(target=formatter)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if errs:
            raise errs[0]
        return total[0]


class FastqFiles:
    """One FASTQ file (unpaired) or the two mate files of paired input (plain or .gz), handed out as engine batches of at most `units`
    reads / pairs: the reader of PatternComposer (pat.cpp) for FASTQ.  The mate files are read in step (bt2g_fastq_parse_pairs_mt
    returns how far it got in each text; the rest waits for the next block), so they need not have lines of equal length."""

    def __init__(self, path1, path2=None, units=500_000, chunk_bytes=64 << 20):
        import gzip
        op = lambda p: gzip.open(p, "rb") if p.endswith(".gz") else open(p, "rb")
        self.f = [op(path1)] + ([op(path2)] if path2 else [])
        self.buf = [b"" for _ in self.f]
        self.eof = [False for _ in self.f]
        self.units, self.chunk = int(units), int(chunk_bytes)

    def _fill(self, k, need_lines):
        while not self.eof[k] and self.buf[k].count(b"\n") < need_lines:
            more = self.f[k].read(self.chunk)
            if not more:
                self.eof[k] = True
                if self.buf[k] and not self.buf[k].endswith(b"\n"):
                    self.buf[k] += b"\n"                         # a last record without a final newline
                break
            self.buf[k] = self.buf[k] + more if self.buf[k] else more

    def next_batch(self, lib, slot, name_stride, threads):
        """-> (ReadBatch, NameTable) of the next batch (mates interleaved), or None at the end of the input"""
        for k in range(len(self.f)):
            self._fill(k, 4 * self.units + 4)
        if len(self.f) == 1:
            if not self.buf[0].strip():
                return None
            batch, names, used = fastq_parse(lib, self.buf[0], max_reads=self.units, name_stride=name_stride, threads=threads, out=slot)
            if batch.n == 0:
                raise RuntimeError("truncated FASTQ record at the end of the input")
            self.buf[0] = self.buf[0][used:]
            self._check_names(names, name_stride)
            return batch, names
        e1, e2 = not self.buf[0].strip(), not self.buf[1].strip()
        if e1 and e2:
            return None
        if e1 or e2:
            # DualPatternComposer::nextBatch (pat.cpp:256-290)
            raise RuntimeError("Error, fewer reads in file specified with -%d than in file specified with -%d" % ((1, 2) if e1 else (2, 1)))
        batch, names, u1, u2 = fastq_parse_pairs(lib, self.buf[0], self.buf[1], name_stride=name_stride, threads=threads, out=slot, max_pairs=self.units)
        if batch.n == 0:
            raise RuntimeError("truncated FASTQ record at the end of the input")
        self.buf[0], self.buf[1] = self.buf[0][u1:], self.buf[1][u2:]
        self._check_names(names, name_stride)
        return batch, names

    @staticmethod
    def _check_names(names, name_stride):
        # the parser keeps name_stride - 1 bytes of a header line: a row filled to its last byte may have lost its tail (the name feeds
        # the read's random seed and the QNAME, so that is an error)
        if len(names) and names.rows[:, name_stride - 2].any():
            raise ValueError(f"a read name is longer than {name_stride - 2} bytes: pass a larger name_stride")

    def close(self):
        for f in self.f:
            f.close()


def align_files_stream(index_base, out_path, reads1, reads2=None, preset="sensitive", local=False, device=0, engines=2, batch_units=500_000,
                       max_read_len=320, name_stride=128, threads=8, seed=0, seed_table=0, dense_sa=-1, offrate=-1, pg_cl=None, summary=None, policy_options=None,
                       gpu=None, make_engine=None):
    """bowtie2 -x index_base (-U reads1 | -1 reads1 -2 reads2) -S out_path through the device engine (bt2g_xengine_*: records identical
    to the reference program's) with the host stages overlapped (TextAligner): file blocks are parsed, aligned by `engines` engines on
    their own streams and host threads, formatted and written in input order.  The primary alignment per read / pair is reported (-M
    mode), or with policy_options {"k": N} / {"all_hits": True} every alignment of -k N / -a: the engines keep up to N entries per read
    (2N + 2 per pair; -a: align.ALL_HITS_CAP / ALL_HITS_CAP_PAIRS, with batch_units cut so that an engine's dense entry arrays stay under
    about 4 GiB, and a warning when a read had more).  policy_options: keyword arguments of lib.policy_params (nofw, norc, mixed,
    discord, pe, sc, mhits, seed_len, k, all_hits ...).  name_stride: bytes kept per read name (a longer header line is an error, not a silent cut).
    Returns the ALIGN_COUNTS record; `summary` (a text stream) receives the alignment summary.
    gpu / make_engine: an open Bt2Gpu with the index loaded / a factory (params, max_units, max_len) -> engine, for callers that keep
    them (and for the CPU tests' stand-ins); under -k / -a it is called with max_per_unit=... as well."""
    from .align import k_caps
    from .lib import ALIGN_COUNTS, Bt2Gpu, IndexFile, XEngine, align_counts_add, align_summary, policy_params, sam_header
    opts = dict(policy_options or {})
    paired = reads2 is not None
    cap, solo_cap = k_caps(opts, paired), k_caps(opts, False)
    if cap is not None:
        # the entry arrays are dense (units x cap rows of a result and an op string, x 2 for pairs): at most ~4 GiB per engine
        row_bytes = 56 + max_read_len + 80 + (12 if paired else 0)
        batch_units = max(1, min(batch_units, (4 << 30) // (cap * (2 if paired else 1) * row_bytes)))
    own = gpu is None
    image = IndexFile(index_base, offrate)
    ref_names, ref_lens = image.ref_names, image.ref_lens
    if own:
        gpu = Bt2Gpu(device)                                     # raises without a GPU: nothing below runs on the CPU
        gpu.load_index_host(image)
        if seed_table:
            gpu.build_seed_table(seed_table)
        if dense_sa >= 0:
            gpu.build_dense_sa(dense_sa)
    image.close()
    lib = load_library()
    prm = policy_params(preset, local=local, paired=paired, seed=seed, host_threads=threads, **opts)
    make_engine = make_engine or (lambda p, n, l, **kw: XEngine(gpu, p, n, l, **kw))
    kcap = (lambda c: {} if c is None else {"max_per_unit": c})
    engs = [make_engine(prm, batch_units, max_read_len, **kcap(cap)) for _ in range(max(1, engines))]
    no_disc, no_mixed = opts.get("discord") is False, opts.get("mixed") is False
    solo_opts = {k: v for k, v in opts.items() if k not in ("pe", "mixed", "discord")}      # the unpaired policy of the same run
    counts = np.zeros(1, dtype=ALIGN_COUNTS)
    src = FastqFiles(reads1, reads2, units=batch_units)
    pthr = max(1, threads // 4)
    ta = TextAligner(engs, [n.split()[0] if n.split() else n for n in ref_names], paired, local=local, parse_threads=pthr,
                     format_threads=max(1, threads - pthr), name_stride=name_stride, no_discordant=no_disc, sc=opts.get("sc"), policy_options=opts,
                     make_solo_engine=(lambda: make_engine(policy_params(preset, local=local, paired=False, seed=seed, host_threads=threads, **solo_opts),
                                                           min(batch_units, 4096), max_read_len, **kcap(solo_cap))) if paired else None)
    try:
        with open(out_path, "wb") as out:
            out.write(sam_header(lib, ref_names, ref_lens, pg_cl).encode())
            ta.run(src, out.write, on_batch=lambda res, pairs: align_counts_add(lib, counts, res, pairs, no_discordant=no_disc))
    finally:
        src.close()
        for e in engs + ([ta._solo] if ta._solo is not None else []):
            if hasattr(e, "close"):
                e.close()
        if own:
            gpu.close()
    if summary is not None:
        summary.write(align_summary(lib, counts, discord=not no_disc, mixed=not no_mixed))
    return counts
