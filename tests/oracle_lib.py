"""ctypes access to the oracle (TEST INFRASTRUCTURE):
  * ``Oracle``    -- oracle/_ref/libbt2oracle.so, the plain-C restatement (oracle/bt2_oracle.c)
  * ``Reference`` -- oracle/_ref/libbt2ref_{s,l}.so, the unmodified reference behind oracle/ref_glue.cpp
Both expose the same method names so tests can run one body against either.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFDIR = os.path.join(ROOT, "oracle", "_ref")
OFFMASK = 0xFFFFFFFFFFFFFFFF

u64, vp, ci = C.c_uint64, C.c_void_p, C.c_int
pu64 = C.POINTER(u64)


def ref_bin(name):
    return os.path.join(REFDIR, name)


def have_reference():
    return os.path.exists(ref_bin("libbt2ref_s.so")) and os.path.exists(ref_bin("bowtie2-build-s"))


def build_oracle():
    """(Re)build the C restatement; also the reference objects when /root/reference is present."""
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "oracle"])
    if os.path.isdir("/root/reference"):
        subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle"), "ref"])


class _Base:
    prefix = ""

    def _bind(self, lib):
        p = self.prefix
        g = lambda n: getattr(lib, p + n)
        g("open").restype = vp; g("open").argtypes = [C.c_char_p, ci, ci]
        g("close").argtypes = [vp]; g("close").restype = None
        g("scalar").restype = u64; g("scalar").argtypes = [vp, ci, ci]
        g("rank4").argtypes = [vp, ci, u64, pu64]; g("rank4").restype = None
        g("rank1").restype = u64; g("rank1").argtypes = [vp, ci, u64, ci]
        g("rowL").restype = ci; g("rowL").argtypes = [vp, ci, u64]
        g("maplf1").restype = u64; g("maplf1").argtypes = [vp, ci, u64, ci]
        g("maplf_range").argtypes = [vp, ci, u64, u64, pu64, pu64, vp]; g("maplf_range").restype = None
        g("ftab_lohi").argtypes = [vp, ci, u64, pu64, pu64]; g("ftab_lohi").restype = None
        g("get_offset").restype = u64; g("get_offset").argtypes = [vp, u64]
        g("get_stretch").argtypes = [vp, u64, C.c_int64, C.c_int64, vp]
        g("exact_sweep").restype = u64
        g("exact_sweep").argtypes = [vp, vp, ci, ci, ci, pu64, pu64]
        g("seed_search").argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, pu64]
        self._g = g

    SCALARS = ["len", "bwt_len", "line_rate", "off_rate", "ftab_chars", "num_sides", "side_sz", "side_bwt_sz",
               "z_off", "n_pat", "n_frag", "offs_len", "ftab_len", "eftab_len", "ebwt_tot_len"]

    def scalars(self, mirror=False):
        return {k: int(self._g("scalar")(self.h, int(mirror), i)) for i, k in enumerate(self.SCALARS)}

    def rank4(self, rows, mirror=False):
        out = np.empty((len(rows), 4), dtype=np.uint64)
        buf = (u64 * 4)()
        for i, r in enumerate(rows):
            self._g("rank4")(self.h, int(mirror), int(r), buf)
            out[i] = list(buf)
        return out

    def maplf1(self, rows, chars, mirror=False):
        return np.array([self._g("maplf1")(self.h, int(mirror), int(r), int(c)) for r, c in zip(rows, chars)], dtype=np.uint64)

    def maplf_range(self, tops, nums, mirror=False):
        """Ebwt::mapLFRange for every [top, top+num): (upto[n,4], in[n,4], chars (one per row, ranges back to back))."""
        upto = np.empty((len(tops), 4), dtype=np.uint64)
        inn = np.empty((len(tops), 4), dtype=np.uint64)
        chars = np.empty(int(np.sum(np.asarray(nums, dtype=np.uint64))), dtype=np.uint8)
        u, n_, o = (u64 * 4)(), (u64 * 4)(), 0
        for i, (t, n) in enumerate(zip(tops, nums)):
            buf = np.empty(int(n), dtype=np.uint8)
            self._g("maplf_range")(self.h, int(mirror), int(t), int(n), u, n_, buf.ctypes.data_as(vp))
            upto[i], inn[i] = list(u), list(n_)
            chars[o:o + int(n)] = buf
            o += int(n)
        return upto, inn, chars

    def ftab_lohi(self, idx, mirror=False):
        out = np.empty((len(idx), 2), dtype=np.uint64)
        t, b = u64(), u64()
        for i, x in enumerate(idx):
            self._g("ftab_lohi")(self.h, int(mirror), int(x), C.byref(t), C.byref(b))
            out[i] = (t.value, b.value)
        return out

    def get_offset(self, rows):
        return np.array([self._g("get_offset")(self.h, int(r)) for r in rows], dtype=np.uint64)

    def joined_to_text(self, qlen, off, reject):
        ti, to, tl, st = u64(), u64(), u64(), ci()
        name = "joined_to_text"
        f = self._g(name)
        f.argtypes = [vp, u64, u64, ci, pu64, pu64, pu64, C.POINTER(ci)]
        ok = f(self.h, int(qlen), int(off), int(reject), C.byref(ti), C.byref(to), C.byref(tl), C.byref(st))
        return ok, ti.value, to.value, tl.value, st.value

    def get_stretch(self, tidx, off, count):
        out = np.empty(count, dtype=np.uint8)
        self._g("get_stretch")(self.h, int(tidx), int(off), int(count), out.ctypes.data_as(vp))
        return out

    def exact_sweep(self, codes, nofw=False, norc=False):
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        m, t = (u64 * 2)(), (u64 * 4)()
        nelt = self._g("exact_sweep")(self.h, codes.ctypes.data_as(vp), len(codes), int(nofw), int(norc), m, t)
        return int(nelt), list(m), list(t)

    def seed_search(self, codes, seed_len, interval, offset, max_seeds, nofw=False, norc=False, quals=None):
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if quals is None:
            quals = np.full(len(codes), ord("I"), dtype=np.uint8)
        quals = np.ascontiguousarray(quals, dtype=np.uint8)
        out = np.zeros((2, max_seeds, 4), dtype=np.uint64)
        n = self._g("seed_search")(self.h, codes.ctypes.data_as(vp), quals.ctypes.data_as(vp), len(codes), seed_len,
                                   interval, offset, int(nofw), int(norc), max_seeds, out.ctypes.data_as(pu64))
        return n, out

    def close(self):
        if self.h:
            self._g("close")(self.h)
            self.h = None


class Oracle(_Base):
    prefix = "bt2o_"

    def __init__(self, base, mirror=True, ref=True):
        path = ref_bin("libbt2oracle.so")
        if not os.path.exists(path):
            build_oracle()
        self.lib = C.CDLL(path)
        self._bind(self.lib)
        self.h = self.lib.bt2o_open(base.encode(), int(mirror), int(ref))
        if not self.h:
            raise RuntimeError(f"oracle: cannot open index {base}")


class Reference(_Base):
    prefix = "ref_"

    def __init__(self, base, mirror=True, ref=True, large=False):
        self.lib = C.CDLL(ref_bin("libbt2ref_l.so" if large else "libbt2ref_s.so"))
        self._bind(self.lib)
        self.h = self.lib.ref_open(base.encode(), int(mirror), int(ref))
        if not self.h:
            raise RuntimeError(f"reference: cannot open index {base}")

    def set_scoring(self, sc):
        """The handle's end-to-end (sc.local False) or local Scoring becomes the one the program builds from a
        bowtie2_b200.policy.Scoring (--ma, --mp with quality-aware mismatches, --np, --rdg, --rfg, the gap barrier, --n-ceil,
        --score-min); ref_dp / ref_ungapped / ref_one_mm use it from then on.  policy.Scoring.default(local) restores the default.

        The reference library is built only where the reference's sources are, and that build is reused elsewhere, so this
        goes through no new glue symbol: it writes the handle's own Scoring object (its plain data members and the three
        penalty tables its constructor fills, _RefScoring) in place.  The layout is checked against the object's own
        invariants before the write and against the reference's Scoring::maxReadGaps / maxRefGaps / perfectScore / nCeil
        (ref_score_params) after it."""
        from bowtie2_b200 import policy
        local = bool(sc.local)
        # RefHandle (oracle/ref_glue.cpp): unique_ptr<Ebwt> fw, bw; unique_ptr<BitPairReference> ref; unique_ptr<Scoring> sc_e2e, sc_loc
        ptr = C.cast(C.c_void_p(self.h + 8 * (4 if local else 3)), C.POINTER(C.c_void_p)).contents.value
        s = _RefScoring.from_address(ptr)
        _RefScoring.check(s)
        smin, nce = sc.score_min(), sc.n_ceil_func()
        s.match_const, s.mmp_max, s.mmp_min, s.npen = sc.match_bonus, sc.mmp_max, sc.mmp_min, sc.n_pen
        s.rd_gap_const, s.rf_gap_const, s.rd_gap_linear, s.rf_gap_linear, s.gapbar = (sc.rdgap_const, sc.rfgap_const, sc.rdgap_linear,
                                                                                   sc.rfgap_linear, sc.gapbar)
        s.monotone = sc.match_bonus == 0
        big = np.finfo(np.float64).max
        s.score_min = _RefSimpleFunc(smin.type, -big, big, float(smin.C), float(smin.L))
        s.n_ceil = _RefSimpleFunc(policy.SIMPLE_FUNC_LINEAR, 0.0, big, float(nce.C), float(nce.L))
        for q in range(256):                                   # Scoring::initPens
            s.mmpens[q] = policy.mm_penalty(q, sc.mmp_max, sc.mmp_min)
            s.npens[q] = sc.n_pen
            s.match_bonuses[q] = float(sc.match_bonus)
        _RefScoring.check(s)
        out4 = np.zeros(4, np.int64)
        f = self.lib.ref_score_params
        f.argtypes = [vp, ci, C.c_int64, u64, vp]
        f.restype = None
        for rdlen in (20, 100, 250):
            minsc = sc.min_score(rdlen)
            f(self.h, int(local), minsc, rdlen, out4.ctypes.data_as(vp))
            want = [sc.max_read_gaps(minsc, rdlen), sc.max_ref_gaps(minsc, rdlen), sc.perfect_score(rdlen), sc.n_ceil_raw(rdlen)]
            if [int(x) for x in out4] != want:
                raise RuntimeError(f"reference Scoring after set_scoring: {list(out4)} != {want} at {rdlen} bp")


class _RefSimpleFunc(C.Structure):
    _fields_ = [("type", ci), ("lo", C.c_double), ("hi", C.c_double), ("const", C.c_double), ("linear", C.c_double)]


class _RefScoring(C.Structure):
    """the data members of the reference's Scoring (scoring.h) up to its penalty tables, in declaration order (no virtual functions:
    the first member is at offset 0)"""
    _fields_ = [("match_type", ci), ("match_const", ci), ("mmcost_type", ci), ("mmp_max", ci), ("mmp_min", ci),
                ("score_min", _RefSimpleFunc), ("n_ceil", _RefSimpleFunc), ("npen_type", ci), ("npen", ci), ("ncatpair", C.c_bool),
                ("rd_gap_const", ci), ("rf_gap_const", ci), ("rd_gap_linear", ci), ("rf_gap_linear", ci), ("gapbar", ci),
                ("monotone", C.c_bool), ("match_bonuses", C.c_float * 256), ("mmpens", ci * 256), ("npens", ci * 256)]
    QUAL, CONSTANT = 2, 3          # COST_MODEL_QUAL, COST_MODEL_CONSTANT

    @staticmethod
    def check(s):
        """the invariants the constructor leaves (quality-aware mismatches, constant N penalty and match bonus, tables filled from
        the scalars): a member at another offset than assumed breaks them"""
        from bowtie2_b200 import policy
        ok = (s.match_type == _RefScoring.CONSTANT and s.mmcost_type == _RefScoring.QUAL and s.npen_type == _RefScoring.CONSTANT
              and s.n_ceil.type == policy.SIMPLE_FUNC_LINEAR and 0 <= s.gapbar < 1 << 16 and s.monotone == (s.match_const == 0)
              and all(s.mmpens[q] == policy.mm_penalty(q, s.mmp_max, s.mmp_min) for q in range(256))
              and all(s.npens[q] == s.npen and s.match_bonuses[q] == s.match_const for q in range(256)))
        if not ok:
            raise RuntimeError("the reference's Scoring object does not have the layout oracle_lib._RefScoring assumes")


# ---- DP through the unmodified SwAligner (oracle/ref_glue_dp.cpp) ------------------------------
def ref_dp(R, local, codes, quals, fw, tidx, tlen, rect, minsc, rndseed=1234, max_cands=1024, max_alns=32, max_edits=4096):
    """Returns dict(found, best, cands[(row,col,score)], alns[dict(score,ns,gaps,refoff,trim5,trim3,fw,edits)])."""
    i64 = C.c_int64
    L = R.lib
    L.ref_dp.argtypes = [vp, ci, vp, vp, ci, ci, u64, i64, C.POINTER(i64), i64, C.c_uint32, ci, ci, ci, vp, vp, vp, vp]
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    quals = np.ascontiguousarray(quals, dtype=np.uint8)
    r9 = (i64 * 9)(rect.refl, rect.refr, rect.refl_pretrim, rect.refr_pretrim, rect.triml, rect.trimr,
                   rect.corel, rect.corer, rect.maxgap)
    summ = np.zeros(4, np.int64)
    cands = np.zeros(3 * max_cands, np.int64)
    alns = np.zeros(8 * max_alns, np.int64)
    eds = np.zeros(4 * max_edits, np.int32)
    L.ref_dp(R.h, int(local), codes.ctypes.data_as(vp), quals.ctypes.data_as(vp), len(codes), int(fw), int(tidx),
             int(tlen), r9, int(minsc), rndseed, max_cands, max_alns, max_edits, summ.ctypes.data_as(vp),
             cands.ctypes.data_as(vp), alns.ctypes.data_as(vp), eds.ctypes.data_as(vp))
    out = {"found": int(summ[0]), "best": int(summ[1]), "ncand": int(summ[2]), "naln": int(summ[3])}
    out["cands"] = [tuple(int(x) for x in cands[3 * i:3 * i + 3]) for i in range(min(out["ncand"], max_cands))]
    al, e0 = [], 0
    for i in range(min(out["naln"], max_alns)):
        a = alns[8 * i:8 * i + 8]
        ne = int(a[6])
        al.append({"score": int(a[0]), "ns": int(a[1]), "gaps": int(a[2]), "refoff": int(a[3]), "trim5": int(a[4]),
                   "trim3": int(a[5]), "fw": int(a[7]),
                   "edits": [[int(x) for x in eds[4 * k:4 * k + 4]] for k in range(e0, e0 + ne)]})
        e0 += ne
    out["alns"] = al
    return out


class _OScoring(C.Structure):
    _fields_ = [(k, C.c_int) for k in ("match_bonus", "mmp_max", "mmp_min", "n_pen", "rdgap_const", "rdgap_linear",
                                       "rfgap_const", "rfgap_linear", "gapbar", "local")] + [("nceil_const", C.c_double), ("nceil_linear", C.c_double)]


SCORING_OVERRIDE = None      # a bowtie2_b200.policy.Scoring: non-default penalties for the oracle calls that follow


def scoring_grid():
    """id -> policy.Scoring: the non-default scorings the DP, ungapped and 1-mismatch kernels are pinned to the reference under.
    Flat and steep mismatch costs (the query profile, quality scaling); N penalties 0 (increments of 0: the edge of the
    "every increment <= 0" arguments of the end-to-end fill) and 3; cheap, asymmetric and const < linear gaps (long gap walks, many
    gap candidates, op strings longer than the read + 64); gap barriers 1 and 10; N ceilings of 0 and half the read; minimum
    scores on both sides of the H-byte limit at 100 bp (1 - minsc <= 127); local with match bonuses 1 and 3 and cheap gaps."""
    from bowtie2_b200 import policy
    F, LIN, LOG = policy.SimpleFunc, policy.SIMPLE_FUNC_LINEAR, policy.SIMPLE_FUNC_LOG
    e2e = {"mp6,6": dict(mmp_max=6, mmp_min=6), "mp2,2": dict(mmp_max=2, mmp_min=2), "mp8,3": dict(mmp_max=8, mmp_min=3),
           "np0": dict(n_pen=0), "np3": dict(n_pen=3), "rdg1,1": dict(rdgap_const=1, rdgap_linear=1), "rfg1,1": dict(rfgap_const=1, rfgap_linear=1),
           "rdg5,1-rfg8,4": dict(rdgap_const=5, rdgap_linear=1, rfgap_const=8, rfgap_linear=4), "rdg3,4": dict(rdgap_const=3, rdgap_linear=4),
           "gapbar1": dict(gapbar=1), "gapbar10": dict(gapbar=10), "nceil-L0,0": dict(n_ceil_over=F(LIN, 0.0, 0.0)),
           "nceil-L0,0.5": dict(n_ceil_over=F(LIN, 0.0, 0.5)), "minsc-126": dict(score_min_func=F(LIN, -126.0, 0.0)),
           "minsc-127": dict(score_min_func=F(LIN, -127.0, 0.0))}
    loc = {"local-ma1": dict(match_bonus=1, rdgap_const=2, rdgap_linear=1, rfgap_const=2, rfgap_linear=1, score_min_func=F(LOG, 10.0, 5.4)),
           "local-ma3": dict(match_bonus=3, rdgap_const=3, rdgap_linear=1, rfgap_const=3, rfgap_linear=1, score_min_func=F(LOG, 20.0, 8.0))}
    out = {k: policy.Scoring(**v) for k, v in e2e.items()}
    out.update({k: policy.Scoring(local=True, **v) for k, v in loc.items()})
    return out


def oracle_scoring(O, local):
    O.lib.bt2o_scoring_default.argtypes = [C.POINTER(_OScoring), ci]
    sc = _OScoring()
    O.lib.bt2o_scoring_default(C.byref(sc), int(local))
    p = SCORING_OVERRIDE
    if p is not None:
        sc.match_bonus, sc.mmp_max, sc.mmp_min, sc.n_pen = p.match_bonus, p.mmp_max, p.mmp_min, p.n_pen
        sc.rdgap_const, sc.rdgap_linear, sc.rfgap_const, sc.rfgap_linear, sc.gapbar = (p.rdgap_const, p.rdgap_linear, p.rfgap_const,
                                                                                        p.rfgap_linear, p.gapbar)
        if p.n_ceil_over is not None:
            sc.nceil_const, sc.nceil_linear = float(p.n_ceil_over.C), float(p.n_ceil_over.L)
    return sc


def oracle_dp(O, local, codes, quals, fw, tidx, rect, minsc, nceil, max_cands=1024, max_alns=32, max_edits=4096, attempts=False):
    """Same outputs as ref_dp(), from the plain-C restatement (oracle/bt2_oracle.c: bt2o_dp).  attempts=True adds
    out["attempts"] = [(candidate score, alignment index or -1)], one entry per backtrace the reference would start."""
    i64 = C.c_int64
    L = O.lib
    att = None
    if attempts:
        att = np.full(3 * 4096, -1, np.int64)
        L.bt2o_dp_attempt_log.argtypes = [vp, ci]
        L.bt2o_dp_attempt_log.restype = None
        L.bt2o_dp_attempt_count.restype = ci
        L.bt2o_dp_attempt_log(att.ctypes.data_as(vp), 4096)
    L.bt2o_scoring_default.argtypes = [C.POINTER(_OScoring), ci]
    L.bt2o_dp.argtypes = [vp, C.POINTER(_OScoring), vp, vp, ci, ci, u64, i64, i64, ci, ci, ci, i64, ci, ci, ci, ci, vp, vp, vp, vp]
    sc = oracle_scoring(O, local)
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    quals = np.ascontiguousarray(quals, dtype=np.uint8)
    summ = np.zeros(4, np.int64)
    cands = np.zeros(3 * max_cands, np.int64)
    alns = np.zeros(8 * max_alns, np.int64)
    eds = np.zeros(4 * max_edits, np.int32)
    L.bt2o_dp(O.h, C.byref(sc), codes.ctypes.data_as(vp), quals.ctypes.data_as(vp), len(codes), int(fw), int(tidx),
              int(rect.refl), int(rect.refr), int(rect.triml), int(rect.corel), int(rect.corer), int(minsc), int(nceil),
              max_cands, max_alns, max_edits, summ.ctypes.data_as(vp), cands.ctypes.data_as(vp), alns.ctypes.data_as(vp),
              eds.ctypes.data_as(vp))
    out = {"found": int(summ[0]), "best": int(summ[1]), "ncand": int(summ[2]), "naln": int(summ[3])}
    out["cands"] = [tuple(int(x) for x in cands[3 * i:3 * i + 3]) for i in range(min(out["ncand"], max_cands))]
    al, e0 = [], 0
    for i in range(min(out["naln"], max_alns)):
        a = alns[8 * i:8 * i + 8]
        ne = int(a[6])
        al.append({"score": int(a[0]), "ns": int(a[1]), "gaps": int(a[2]), "refoff": int(a[3]), "trim5": int(a[4]),
                   "trim3": int(a[5]), "fw": int(a[7]),
                   "edits": [[int(x) for x in eds[4 * k:4 * k + 4]] for k in range(e0, e0 + ne)]})
        e0 += ne
    out["alns"] = al
    if attempts:
        n = int(L.bt2o_dp_attempt_count())
        assert n <= 4096
        out["attempts"] = [(int(att[3 * k]), int(att[3 * k + 1])) for k in range(n)]
        out["attempt_cands"] = [int(att[3 * k + 2]) for k in range(n)]
        L.bt2o_dp_attempt_log(None, 0)
    return out


def extend_both(X, codes, fw, off, seedlen, rng4):
    """SwDriver::extend through the reference glue (X = Reference) or the C restatement (X = Oracle)."""
    out = (u64 * 2)()
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    f = X._g("extend")
    f.argtypes = [vp, vp, ci, ci, u64, u64, u64, u64, u64, u64, pu64]
    f.restype = None
    f(X.h, codes.ctypes.data_as(vp), len(codes), int(fw), int(off), int(seedlen), int(rng4[0]), int(rng4[1]), int(rng4[2]), int(rng4[3]), out)
    return int(out[0]), int(out[1])


# ---- SeedAligner::oneMmSearch (oracle/ref_glue.cpp: ref_one_mm, oracle/bt2_oracle.c: bt2o_one_mm) ----
def _one_mm_call(fn, first, codes, quals, minsc, nofw, norc, max_hits):
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    if quals is None:
        quals = np.full(len(codes), ord("I"), dtype=np.uint8)
    quals = np.ascontiguousarray(quals, dtype=np.uint8)
    out = np.zeros((max_hits, 6), dtype=np.int64)
    fws = np.zeros(max_hits, dtype=np.int32)
    fn.restype = ci
    n = fn(*first, codes.ctypes.data_as(vp), quals.ctypes.data_as(vp), ci(len(codes)), C.c_int64(int(minsc)),
           ci(int(nofw)), ci(int(norc)), ci(max_hits), out.ctypes.data_as(vp), fws.ctypes.data_as(vp))
    assert n <= max_hits
    return [tuple(int(x) for x in out[i]) + (int(fws[i]),) for i in range(n)]


def ref_one_mm(R, local, codes, quals, minsc, nofw=False, norc=False, max_hits=256):
    """-> list of (top, bot, pos, chr, qchr, score, fw) in SeedResults::mm1EEHits() order."""
    return _one_mm_call(R.lib.ref_one_mm, (vp(R.h), ci(int(local))), codes, quals, minsc, nofw, norc, max_hits)


def oracle_one_mm(O, local, codes, quals, minsc, nofw=False, norc=False, max_hits=256):
    sc = oracle_scoring(O, local)
    return _one_mm_call(O.lib.bt2o_one_mm, (vp(O.h), C.byref(sc)), codes, quals, minsc, nofw, norc, max_hits)


# ---- SwAligner::ungappedAlign (oracle/ref_glue_dp.cpp: ref_ungapped, oracle/bt2_oracle.c: bt2o_ungapped) ----
def ref_ungapped(R, local, codes, quals, fw, tidx, off, tlen, ohang, minsc, max_edits=1024):
    """-> (rc, dict(score, refoff, trim5, trim3, ns, refns, edits=[(pos, chr, qchr, type)]))"""
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    quals = np.ascontiguousarray(quals, dtype=np.uint8)
    out8 = np.zeros(8, np.int64)
    ed = np.zeros(4 * max_edits, np.int32)
    f = R.lib.ref_ungapped
    f.restype = ci
    i64 = C.c_int64
    rc = f(vp(R.h), ci(int(local)), codes.ctypes.data_as(vp), quals.ctypes.data_as(vp), ci(len(codes)), ci(int(fw)), u64(int(tidx)),
           i64(int(off)), i64(int(tlen)), ci(int(ohang)), i64(int(minsc)), ci(max_edits), out8.ctypes.data_as(vp), ed.ctypes.data_as(vp))
    n = int(out8[6])
    return rc, dict(score=int(out8[0]), refoff=int(out8[1]), trim5=int(out8[2]), trim3=int(out8[3]), ns=int(out8[4]),
                    refns=int(out8[5]), edits=[tuple(int(x) for x in ed[4 * k:4 * k + 4]) for k in range(n)])


def oracle_ungapped(O, local, codes, quals, fw, tidx, off, tlen, ohang, minsc):
    """-> (rc, dict(score, rowi, rowf, ns, refns, nedits, mask))"""
    sc = oracle_scoring(O, local)
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    quals = np.ascontiguousarray(quals, dtype=np.uint8)
    out6 = np.zeros(6, np.int64)
    mask = np.zeros(len(codes), np.uint8)
    f = O.lib.bt2o_ungapped
    f.restype = ci
    i64 = C.c_int64
    rc = f(vp(O.h), C.byref(sc), codes.ctypes.data_as(vp), quals.ctypes.data_as(vp), ci(len(codes)), ci(int(fw)), u64(int(tidx)),
           i64(int(off)), i64(int(tlen)), ci(int(ohang)), i64(int(minsc)), out6.ctypes.data_as(vp), mask.ctypes.data_as(vp))
    return rc, dict(score=int(out6[0]), rowi=int(out6[1]), rowf=int(out6[2]), ns=int(out6[3]), refns=int(out6[4]),
                    nedits=int(out6[5]), mask=mask)


def oracle_policy_table(O, local=False, off_size=4, scoring=None):
    """bt2g_policy_backend filled with the C oracle's functions (oracle/bt2_oracle_table.c): the exact-policy engine driven on the
    CPU at C speed.  Returns (table, handle to keep alive)."""
    from bowtie2_b200.lib import _PolicyBackend
    be = _PolicyBackend()
    O.lib.bt2o_policy_table.argtypes = [vp, ci, ci, C.POINTER(_PolicyBackend)]
    O.lib.bt2o_policy_table.restype = vp
    h = O.lib.bt2o_policy_table(O.h, int(local), int(off_size), C.byref(be))
    if scoring is not None:
        O.lib.bt2o_policy_table_scoring.argtypes = [vp] + [ci] * 8
        O.lib.bt2o_policy_table_scoring.restype = None
        O.lib.bt2o_policy_table_scoring(h, scoring.match_bonus, scoring.mmp_max, scoring.mmp_min, scoring.n_pen, scoring.rdgap_const,
                                        scoring.rdgap_linear, scoring.rfgap_const, scoring.rfgap_linear)
        if scoring.n_ceil_over is not None:
            O.lib.bt2o_policy_table_nceil.argtypes = [vp, C.c_double, C.c_double]
            O.lib.bt2o_policy_table_nceil.restype = None
            O.lib.bt2o_policy_table_nceil(h, float(scoring.n_ceil_over.C), float(scoring.n_ceil_over.L))
    return be, (O, h)
