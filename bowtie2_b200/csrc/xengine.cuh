// xengine.cuh -- the reference's sequential, RNG-driven search policy for PAIRS and single reads (multiseedSearchWorker,
// bt2_search.cpp:3094-4254; SwDriver::extendSeeds / extendSeedsPaired, aligner_sw_driver.cpp:921-2637; AlnSinkWrap /
// ReportingState, aln_sink.cpp) as an explicit, fixed-memory STATE MACHINE that compiles for the host and for the device.
//
// csrc/policy_engine.cpp holds the same policy as C++20 coroutines over heap containers (pinned byte-for-byte against the
// reference program's SAM); this file is its device-shaped twin: one `XUnit` per read pair (or read) in HBM, every container a
// fixed-capacity array or a bump-allocated arena inside the unit, control flow as a protothread (switch on a saved program
// counter) that runs until it needs a BATCHED primitive -- a DP problem, a mate-finding DP problem, a 1-mismatch search or a
// seed search -- and returns that request to its caller.  The cheap primitives (SA-offset resolution, SwDriver::extend,
// ungapped alignment) are called inline through the `Svc` template parameter.  On the GPU the caller is k_xe_step (one thread
// per unit, csrc/xengine.cu) and the requests go to device queues consumed by the DP / FM kernels once per wave; on the CPU
// (csrc/xengine_host.cpp) the caller answers each request at once through the bt2g_policy_backend table, which is how this
// file is pinned against the reference program in the CPU test-suite.
//
// A unit that outgrows a capacity (arena, lists) stops with XR_FALLBACK and is re-run by the coroutine engine
// (bt2g_policy_align over the same device primitives): capacities bound memory, never results.
#pragma once
#include <stdint.h>
#include "../../include/bt2g.h"
#include "mapq_device.cuh"
#include "pe_device.cuh"

#ifndef XE_HD
#define XE_HD __host__ __device__
#endif
#define XE_HH __host__ __device__      // always both: the parameter arithmetic is also used by the host-side set-up

namespace xe {

// ---------------------------------------------------------------------------------------------- constants
#define XE_MIN_I64 (-9223372036854775807LL - 1)
#define XE_BIG ((int64_t)1 << 62)
enum { EXHAUSTED = 1, FULFILLED, PERFECT, SOFT_LIMIT, HARD_LIMIT };
// what a step returns: 0 = finished; otherwise the batched primitive the unit now waits for
enum { XR_DONE = 0, XR_ONE_MM = 1, XR_SEED = 2, XR_DP = 3, XR_DP_MATE = 4, XR_FALLBACK = 5 };

#define XE_MAX_LEN    512
#define XE_ARENA      12288      // bytes
#define XE_SEEN_IV    224        // seenDiags intervals per mate (two per framed DP)
#define XE_EXR        8          // seedExRange entries per mate and strand
#define XE_MM1        24         // 1-mismatch end-to-end hits kept per mate
#define XE_MAX_SEEDS  64         // seed offsets per strand
#define XE_SATS       (2 * XE_MAX_SEEDS)
#define XE_ENTS       416        // satpos entries (<= maxIters + 1)
#define XE_RANDS      160        // Random1toN states of multi-element entries
#define XE_SEENPOOL   416        // pooled "seen" draws of the non-swap-list Random1toN states
#define XE_LIST       64         // alignments per sink list
#define XE_RED        176        // alignments per redundancy set (a pair stopping after mhits + 1 = 51 concordant placements adds 2 x 51 to set 0)
#define XE_ATT        256        // backtrace attempts kept of the anchor DP
#define XE_HITL       (2 + XE_MM1)

// a unit that outgrows a capacity: remember where (line of this file) and stop at the next check
#define XE_FB(U) ((U).fbLine = (U).fallback ? (U).fbLine : (uint32_t)__LINE__, (U).fallback = 1)

// ---------------------------------------------------------------------------------------------- parameters
struct XParams {
	int32_t local, paired, mmode, all, nofw, norc, discord, mixed;
	int32_t seedLen, seedRounds, streak, maxIters, maxUg, maxDp, maxMateStreak;
	int64_t khits, mhits;
	uint32_t seed; int32_t offSize;
	int32_t matchBonus, mmpMax, mmpMin, nPen, rdgConst, rdgLin, rfgConst, rfgLin;
	bt2g_pe_policy pe;
	int32_t maxLen;                                     // tables below hold maxLen + 1 entries
	const int32_t *minscTab, *nceilRawTab, *ivalOneTab, *ivalBothTab;   // SimpleFunc values per read length (host-evaluated doubles)
	XE_HH int64_t perfect(int len) const { return (int64_t)len * matchBonus; }
	XE_HH int64_t minScore(int len) const { return minscTab[len]; }
	XE_HH int nCeilRaw(int len) const { return nceilRawTab[len]; }
	XE_HH int nCeil(int len) const { const int r = nceilRawTab[len]; return r < len ? r : len; }
	XE_HH int seedInterval(int len, bool both) const { return both ? ivalBothTab[len] : ivalOneTab[len]; }
	XE_HH int maxReadGaps(int64_t minsc, int len) const {       // Scoring::maxReadGaps (scoring.cpp:42-66)
		int64_t sc = perfect(len); bool first = true; int num = 0;
		while(sc >= minsc) { sc -= first ? rdgConst + rdgLin : rdgLin; first = false; num++; }
		return num - 1;
	}
	XE_HH int maxRefGaps(int64_t minsc, int len) const {        // Scoring::maxRefGaps (scoring.cpp:73-98)
		int64_t sc = perfect(len); bool first = true; int num = 0;
		while(sc >= minsc) { sc -= matchBonus; sc -= first ? rfgConst + rfgLin : rfgLin; first = false; num++; }
		return num - 1;
	}
	XE_HH int mmPenalty(int q) const { const int ii = q < 0 ? 0 : (q > 40 ? 40 : q); const float frac = (float)ii / 40.0f; return mmpMin + (int)(frac * (float)(mmpMax - mmpMin)); }
};

// ---------------------------------------------------------------------------------------------- small pieces
struct XRng {                                        // RandomSource (random_source.h:32-180)
	uint32_t last; int32_t lastOff;
	XE_HD void init(uint32_t s) { last = s; lastOff = 30; }
	XE_HD uint32_t u32() {
		last = 1664525u * last + 1013904223u;
		uint32_t ret = last >> 16;
		last = 1664525u * last + 1013904223u;
		ret ^= last;
		lastOff = 0;
		return ret;
	}
	XE_HD uint64_t u64() { const uint64_t hi = u32(); return (hi << 32) | u32(); }
	XE_HD int boolean() { if(lastOff > 31) u32(); const int r = (last >> lastOff) & 1; lastOff++; return r; }
	XE_HD double flt() { return (double)((float)u32() / (float)0xffffffff); }
};

struct XEdit { int16_t pos; uint8_t chr, qchr, type, pad; };      // type 1 read gap, 2 ref gap, 3 mismatch; chr / qchr ASCII, '-' for gaps
// alignment record in the unit's arena; edits are kept LEFT TO RIGHT on the reference strand (AlnRes::invertEdits applied once)
struct XAln {
	int64_t refoff; int32_t tidx, score; int16_t rdlen, trim5, trim3, nedits; uint8_t fw, ns, refns, pad;
	XE_HD XEdit *edits() { return reinterpret_cast<XEdit *>(this + 1); }
	XE_HD const XEdit *edits() const { return reinterpret_cast<const XEdit *>(this + 1); }
	XE_HD int ext() const { return rdlen - trim5 - trim3; }
	XE_HD int trimLeft() const { return fw ? trim5 : trim3; }
	XE_HD int refExtent() const { int e = ext(); const XEdit *ed = edits(); for(int i = 0; i < nedits; i++) e += (ed[i].type == 1) - (ed[i].type == 2); return e; }
};

struct XEEHit { uint64_t top, bot; int32_t score; int16_t pos; uint8_t fw, hasEdit, chr, qchr, pad[2];
	XE_HD int ns() const { return hasEdit && (chr == 'N' || qchr == 'N'); }
	XE_HD int refns() const { return hasEdit && chr == 'N'; } };

struct XIv { int64_t a; int32_t tidx, len; };        // tidx: bit 31 = fw
struct XExr { int32_t p5, len; int64_t size; };

struct XRand {                                       // Random1toN (random_util.h:32-160); list / seen storage lives in the unit
	uint32_t n, cur, thresh; uint16_t listOff; uint8_t swaplist, converted;
};
struct XSeen { uint32_t val; uint16_t owner, pad; };

struct XSat { uint64_t topf, topb; int64_t size; int16_t rdoff, seedlen; uint8_t fw, offidx, nlex, nrex; uint8_t rix, elim, pad[2]; double mass; };
struct XEnt { uint64_t topf; int32_t size; int16_t rdoff, seedlen; uint8_t fw; int8_t ee; uint8_t rix, done1, mateStreak, pad[3]; };

struct XMate {
	int32_t idx, rdlen, nceil; int64_t minsc, perfect;
	uint8_t filt, nee, nmm1, hasSh; uint8_t nexr[2]; uint16_t nseen;
	XEEHit ee[2], mm1[XE_MM1];
	XExr exr[2][XE_EXR];
	XIv seen[XE_SEEN_IV];
	int32_t shN, shInterval, shOffset, shSeedlen; int64_t shNonz, shNelt;
	uint16_t nranks; uint8_t ranks[2 * XE_MAX_SEEDS];    // offidx | (fw << 7)
};

struct XDpReq { bt2g_dp_problem prob; };

struct XUnit {
	// ---- protothread state
	int32_t pc, pcExt; uint8_t fallback, paired, doneFlag, pad0;
	uint32_t id;                                          // pair / read index in the batch
	XRng rnd;
	XMate m[2]; int32_t cur;
	// ---- sinks
	int64_t khits, mhits;
	// paired sink
	uint8_t doneConcord, doneDiscord, doneUnp[2], exitConcordM, exitConcordK, psDone, pad1;
	int64_t nconcord, nunp[2], bestPair, best2Pair;
	uint16_t nrs12, nrs1u, nrs2u; uint16_t rs1[XE_LIST], rs2[XE_LIST], rs1u[XE_LIST], rs2u[XE_LIST];
	// unpaired sink
	uint8_t usDone, usExitM, usExitK, pad2; int64_t usBest, usBest2; uint16_t nus; uint16_t usAlns[XE_LIST];
	// redundancy sets: 0 = red, 1 / 2 = redMate[0 / 1]
	uint16_t nred[3]; uint16_t red[3][XE_RED];
	uint32_t redKey[3][XE_RED];                           // coarse locus of each entry (x_red_key): the scan skips far-away entries without touching them
	int64_t nIters, nDps, nUgs, nMateDps, streakCur;
	// ---- pairSteps / readSteps locals
	int32_t interval[2], nrounds[2], matemap[2], mi, roundi, nroundsAll; int64_t nelt[2]; int32_t mined[2][2];
	uint8_t done[2], nofwM[2], norcM[2], both, rdone;
	// ---- extendSeeds[Paired] arguments and locals
	int32_t xAi, xUseSh, xUseEe, xRet;
	uint8_t eeMode, firstEe, firstExtend, swMateImmediately;
	int64_t nEeFail, nUgFail, nDpFail, neltLeft, streak, nonz;
	int32_t si, nents; XEnt ents[XE_ENTS];
	int32_t nsats; XSat sats[XE_SATS];
	int32_t nrands; XRand rands[XE_RANDS];
	int32_t nseenPool; XSeen seenPool[XE_SEENPOOL];
	int32_t nhitl; XEEHit hitl[XE_HITL];
	// iteration locals
	uint8_t isSmall, fw, first, state, firstInner, foundConcordant, foundMate, didAnchor, brk, haveOa, oleft, ofw, dpU8, odpU8, pad3[2];
	int32_t rdoff, readGaps, refGaps;
	int64_t tidx, toff, tlen, refoff, ominscCur;
	uint16_t fixedAln, curAln;                            // arena offsets
	// anchor DP attempts
	int32_t natt, attCursor; int16_t attScore[XE_ATT]; uint16_t attAln[XE_ATT];
	int32_t mateCursor, mateAlnK;                         // cursor into the mate DP's candidate list / alignment list
	// ---- request to the caller (valid when a step returns != XR_DONE)
	bt2g_dp_problem rqProb;                               // XR_DP / XR_DP_MATE
	int32_t rqRead, rqMinsc, rqNofw, rqNorc, rqL, rqInterval, rqOffset;   // XR_ONE_MM / XR_SEED
	int32_t dpSlot;                                       // written by the caller: where the answer of the pending request is
	// ---- result (finishPair / finishRead)
	int32_t pairType, pairKind; int64_t scoreSum, fraglen;
	uint8_t resAligned[2], resHasXs[2]; int32_t resMapq[2]; int64_t resXs[2]; uint16_t resAln[2];
	// ---- arena
	uint32_t arenaTop; uint32_t fbLine;                   // fbLine: source line of the capacity that stopped the unit (diagnostics)
	alignas(8) uint8_t arena[XE_ARENA];
};

// ---------------------------------------------------------------------------------------------- arena helpers
XE_HD inline XAln *x_aln(XUnit &u, uint16_t off) { return reinterpret_cast<XAln *>(u.arena + (size_t)off * 8); }
XE_HD inline const XAln *x_aln(const XUnit &u, uint16_t off) { return reinterpret_cast<const XAln *>(u.arena + (size_t)off * 8); }
// allocate `bytes` (rounded up to 8); returns the offset in 8-byte units, or 0xffff and sets u.fallback
XE_HD inline uint16_t x_alloc(XUnit &u, uint32_t bytes) {
	const uint32_t need = (bytes + 7u) & ~7u;
	if(u.arenaTop + need > XE_ARENA) { XE_FB(u); return 0xffff; }
	const uint16_t off = (uint16_t)(u.arenaTop >> 3);
	u.arenaTop += need;
	return off;
}
XE_HD inline uint16_t x_new_aln(XUnit &u, int nedits) {
	const uint16_t off = x_alloc(u, (uint32_t)(sizeof(XAln) + (size_t)nedits * sizeof(XEdit)));
	if(off == 0xffff) return off;
	XAln *a = x_aln(u, off);
	a->refoff = 0; a->tidx = 0; a->score = 0; a->rdlen = 0; a->trim5 = a->trim3 = 0; a->nedits = (int16_t)nedits; a->fw = 1; a->ns = a->refns = a->pad = 0;
	return off;
}

XE_HD inline char x_dna(int c) { return c == 0 ? 'A' : c == 1 ? 'C' : c == 2 ? 'G' : c == 3 ? 'T' : 'N'; }
XE_HD inline int x_code(int ch) { return ch == 'A' ? 0 : ch == 'C' ? 1 : ch == 'G' ? 2 : ch == 'T' ? 3 : 4; }
XE_HD inline int x_rdchar(const uint8_t *codes, int rdlen, bool fw, int row) {    // strand-oriented read character code
	if(fw) return codes[row];
	const int c = codes[rdlen - 1 - row];
	return c > 3 ? 4 : 3 - c;
}

// ---------------------------------------------------------------------------------------------- Random1toN
XE_HD inline uint16_t *x_rlist(XUnit &u, const XRand &r) { return reinterpret_cast<uint16_t *>(u.arena + (size_t)r.listOff * 8); }
XE_HD inline void x_rand_init(XUnit &u, XRand &r, uint64_t n, bool all) {
	r.n = (uint32_t)n; r.cur = 0; r.converted = 0; r.swaplist = (n < 128 || all) ? 1 : 0; r.listOff = 0xffff;
	const uint32_t t = (uint32_t)(0.10f * (float)n);
	r.thresh = t > 16 ? t : 16;
	if(n > 60000) { if(r.swaplist) XE_FB(u); }          // (-a mode on huge ranges: coroutine engine)
}
XE_HD inline bool x_rand_done(const XRand &r) { return r.n > 0 && r.cur >= r.n; }
XE_HD inline uint32_t x_rand_next(XUnit &u, int rix, XRng &rnd) {
	XRand &r = u.rands[rix];
	if(r.cur == 0 && !r.converted) {
		if(r.n == 1) { r.cur = 1; return 0; }
		if(r.swaplist) {
			r.listOff = x_alloc(u, r.n * 2u);
			if(r.listOff == 0xffff) { r.cur = r.n; return 0; }
			uint16_t *l = x_rlist(u, r);
			for(uint32_t i = 0; i < r.n; i++) l[i] = (uint16_t)i;
		}
	}
	if(r.swaplist) {
		uint16_t *l = x_rlist(u, r);
		const uint32_t k = r.cur + (rnd.u32() % (r.n - r.cur));
		if(k != r.cur) { const uint16_t t = l[r.cur]; l[r.cur] = l[k]; l[k] = t; }
		return l[r.cur++];
	}
	// seen-list mode (n >= 128): draw until unseen
	uint32_t rn;
	for(;;) {
		rn = rnd.u32() % r.n;
		bool again = false;
		for(int i = 0; i < u.nseenPool; i++) if(u.seenPool[i].owner == (uint16_t)rix && u.seenPool[i].val == rn) { again = true; break; }
		if(!again) break;
	}
	if(u.nseenPool >= XE_SEENPOOL) { XE_FB(u); r.cur = r.n; return rn; }
	u.seenPool[u.nseenPool].val = rn; u.seenPool[u.nseenPool].owner = (uint16_t)rix; u.nseenPool++;
	r.cur++;
	uint32_t mine = 0;
	for(int i = 0; i < u.nseenPool; i++) mine += u.seenPool[i].owner == (uint16_t)rix;
	if(mine >= r.thresh && r.cur < r.n) {
		// convert to a swap list of the unseen elements, ascending (random_util.h:118-145)
		const uint32_t rest = r.n - mine;
		if(r.n > 65535u) { XE_FB(u); r.cur = r.n; return rn; }
		r.listOff = x_alloc(u, rest * 2u);
		if(r.listOff == 0xffff) { r.cur = r.n; return rn; }
		uint16_t *l = x_rlist(u, r);
		uint32_t k = 0;
		for(uint32_t j = 0; j < r.n; j++) {
			bool s = false;
			for(int i = 0; i < u.nseenPool; i++) if(u.seenPool[i].owner == (uint16_t)rix && u.seenPool[i].val == j) { s = true; break; }
			if(!s) l[k++] = (uint16_t)j;
		}
		// drop this owner's seen entries
		int w = 0;
		for(int i = 0; i < u.nseenPool; i++) if(u.seenPool[i].owner != (uint16_t)rix) u.seenPool[w++] = u.seenPool[i];
		u.nseenPool = w;
		r.cur = 0; r.n = rest; r.converted = 1; r.swaplist = 1;
	}
	return rn;
}
XE_HD inline int x_new_rand(XUnit &u, uint64_t n, bool all) {
	if(u.nrands >= XE_RANDS) { XE_FB(u); return 0; }
	const int rix = u.nrands++;
	x_rand_init(u, u.rands[rix], n, all);
	return rix;
}

// shuffles over small index arrays (EList::shufflePortion, ds.h; used by selectByScore and eeSaTups)
template <typename T>
XE_HD inline void x_shuffle_portion(T *v, int begin, int num, XRng &rnd) {
	if(num < 2) return;
	int left = num;
	for(int i = begin; i < begin + num - 1; i++) {
		const int r = (int)(rnd.u64() % (uint64_t)left);
		if(r > 0) { const T t = v[i]; v[i] = v[i + r]; v[i + r] = t; }
		left--;
	}
}

// ---------------------------------------------------------------------------------------------- seenDiags / redundancy
XE_HD inline void x_seen_add(XUnit &u, XMate &c, int64_t tidx, bool fw, int64_t off, int64_t len) {
	if(c.nseen >= XE_SEEN_IV) { XE_FB(u); return; }
	XIv &x = c.seen[c.nseen++];
	x.a = off; x.len = (int32_t)len; x.tidx = (int32_t)((uint32_t)tidx | (fw ? 0x80000000u : 0u));
}
XE_HD inline bool x_seen_present(const XMate &c, int64_t tidx, bool fw, int64_t off) {
	const int32_t key = (int32_t)((uint32_t)tidx | (fw ? 0x80000000u : 0u));
	for(int i = 0; i < c.nseen; i++) { const XIv &x = c.seen[i]; if(x.tidx == key && x.a <= off && off < x.a + x.len) return true; }
	return false;
}

// RedundantAlns (aligner_result.cpp:929-1030): the cells an alignment passes through; two alignments are redundant when they
// share a cell.  The reference hashes the cells; here the stored alignments themselves are the set and membership is tested
// by walking both alignments row by row.
struct XCellIt {                                     // per read row: reference columns [left, right)
	const XAln *a; const XEdit *ed; int k, i, n; int64_t left, right, diff;
	XE_HD void init(const XAln *al) { a = al; ed = al->edits(); k = 0; i = al->trimLeft(); n = i + al->ext(); left = al->refoff; right = left + 1; diff = 1; fetch(); }
	XE_HD bool valid() const { return i < n; }
	XE_HD void fetch() {
		if(i >= n) return;
		diff = 1; right = left + 1;
		const int rel = i - a->trimLeft();
		while(k < a->nedits && ed[k].pos == rel) { if(ed[k].type == 2) diff = 0; k++; }
		if(i < n - 1) { int k2 = k; while(k2 < a->nedits && ed[k2].pos == rel + 1) { if(ed[k2].type == 1) right++; k2++; } }
	}
	XE_HD void next() { left = right + diff - 1; i++; fetch(); }
};
XE_HD inline bool x_alns_share_cell(const XAln *a, const XAln *b) {
	if(a->tidx != b->tidx || a->fw != b->fw) return false;
	const int64_t d = a->refoff - b->refoff;
	if(d > 1200 || d < -1200) return false;
	XCellIt x, y; x.init(a); y.init(b);
	while(x.valid() && y.valid()) {
		if(x.i < y.i) { x.next(); continue; }
		if(y.i < x.i) { y.next(); continue; }
		if(x.left < y.right && y.left < x.right) return true;
		x.next(); y.next();
	}
	return false;
}
// NOTE on positions: XEdit.pos is relative to the first aligned read character in left-to-right order (= Edit.pos after
// invertEdits), rows i run over trimLeft .. trimLeft + ext - 1 as in RedundantAlns::add.
// coarse locus of an alignment: 12 bits of (reference, strand), 20 bits of refoff / 2048.  Two alignments that share a cell lie on the
// same reference and strand within 1200 positions of each other (x_alns_share_cell), i.e. in the same or neighbouring buckets.
XE_HD inline uint32_t x_red_key(const XAln *a) {
	return (((uint32_t)a->tidx * 2u + (uint32_t)(a->fw != 0)) << 20) | ((uint32_t)((uint64_t)a->refoff >> 11) & 0xfffffu);
}
XE_HD inline bool x_red_overlap(const XUnit &u, int set, uint16_t aoff) {
	const XAln *a = x_aln(u, aoff);
	const uint32_t ka = x_red_key(a);
	for(int i = 0; i < u.nred[set]; i++) {
		const uint32_t kb = u.redKey[set][i];
		if((ka ^ kb) >> 20) continue;                                   // another reference or strand (or a hash neighbour: checked below)
		if(((kb - ka + 1u) & 0xfffffu) > 2u) continue;                  // buckets further apart than one
		if(x_alns_share_cell(a, x_aln(u, u.red[set][i]))) return true;
	}
	return false;
}
XE_HD inline void x_red_add(XUnit &u, int set, uint16_t aoff) {
	if(u.nred[set] >= XE_RED) { XE_FB(u); return; }
	u.redKey[set][u.nred[set]] = x_red_key(x_aln(u, aoff));
	u.red[set][u.nred[set]++] = aoff;
}

// ---------------------------------------------------------------------------------------------- DP framing
struct XRect { int64_t refl, refr, reflPre, refrPre, triml, trimr, corel, corer, maxgap; };
XE_HD inline bool x_frame_seed(int64_t off, int rdlen, int64_t reflen, int maxrdgap, int maxrfgap, int maxhalf, XRect &r) {
	// DynProgFramer::frameSeedExtensionRect (dp_framer.cpp:81-129); the gap counts are size_t there: negative wraps to huge
	const uint64_t a = (uint64_t)(int64_t)maxrdgap, b = (uint64_t)(int64_t)maxrfgap;
	const uint64_t mx = a > b ? a : b;
	const int64_t maxgap = (int64_t)(mx < (uint64_t)maxhalf ? mx : (uint64_t)maxhalf);
	const int64_t refl = off - 2 * maxgap, refr = off + (rdlen - 1) + 2 * maxgap;
	int64_t triml = 0, trimr = 0;
	if(refr >= reflen) trimr = refr - (reflen - 1);
	if(refl < 0) triml = -refl;
	r.refl = refl + triml; r.refr = refr - trimr; r.reflPre = refl; r.refrPre = refr; r.triml = triml; r.trimr = trimr;
	r.corel = maxgap; r.corer = maxgap + 2 * maxgap; r.maxgap = maxgap;
	return !(r.refr < r.refl);
}
XE_HD inline bool x_frame_mate(bool anchorLeft, int64_t ll, int64_t lr, int64_t rl, int64_t rr, int rdlen, int64_t reflen, int maxrdgap, int maxrfgap,
                               int maxhalf, XRect &r) {
	// DynProgFramer::frameFindMateRect (dp_framer.cpp:177-361): maxgap = max(gaps, maxhalf)
	const uint64_t a = (uint64_t)(int64_t)maxrdgap, b = (uint64_t)(int64_t)maxrfgap;
	uint64_t mx = a > b ? a : b; if((uint64_t)maxhalf > mx) mx = (uint64_t)maxhalf;
	const int64_t maxgap = (int64_t)mx;
	int64_t refl, refr;
	if(anchorLeft) { refl = (rl - (rdlen - 1)) - maxgap; refr = rr + maxgap; }
	else { refl = ll - maxgap; refr = (lr + (rdlen - 1)) + maxgap; }
	int64_t triml = 0, trimr = 0;
	if(refr >= reflen) trimr = refr - (reflen - 1);
	if(refl < 0) triml = -refl;
	const int64_t width = refr - refl + 1;
	r.refl = refl + triml; r.refr = refr - trimr; r.reflPre = refl; r.refrPre = refr; r.triml = triml; r.trimr = trimr;
	r.corel = maxgap; r.corer = width - maxgap - 1; r.maxgap = maxgap;
	return !(r.refr < r.refl);
}

// ---------------------------------------------------------------------------------------------- alignments from primitives
// device op string (include/bt2g.h: bt2g_dp_aln) -> arena record with left-to-right edits (lib.py: ops_to_edits without the
// final inversion for reverse-strand reads)
XE_HD inline uint16_t x_aln_from_dp(XUnit &u, const bt2g_dp_problem &prob, const bt2g_dp_aln &al, const uint8_t *ops, const uint8_t *codes, int rdlen) {
	// one pass: the record is allocated for the largest edit list the op string can hold (every op an edit) and the unused
	// tail of that allocation -- the arena's newest -- is given back
	const uint16_t off = x_new_aln(u, al.nops);
	if(off == 0xffff) return off;
	XAln *a = x_aln(u, off);
	const bool fw = prob.fw != 0;
	a->tidx = (int32_t)prob.tidx; a->refoff = prob.refl + al.col0; a->fw = fw; a->score = al.score; a->rdlen = (int16_t)rdlen;
	a->ns = (uint8_t)al.ns; a->refns = (uint8_t)al.refns;
	a->trim5 = (int16_t)(fw ? al.trim_beg : al.trim_end); a->trim3 = (int16_t)(fw ? al.trim_end : al.trim_beg);
	XEdit *ed = a->edits();
	int row = al.row0, n = 0;
	for(int k = al.nops - 1; k >= 0; k--) {
		const int typ = ops[k] & 3, refc = (ops[k] >> 2) & 7;
		if(typ == BT2G_OP_MATCH) { row++; continue; }
		XEdit &e = ed[n++];
		e.pos = (int16_t)(row - al.row0); e.pad = 0;
		if(typ == BT2G_OP_MM) { e.chr = (uint8_t)x_dna(refc); e.qchr = (uint8_t)x_dna(x_rdchar(codes, rdlen, fw, row)); e.type = 3; row++; }
		else if(typ == BT2G_OP_REFGAP) { e.chr = '-'; e.qchr = (uint8_t)x_dna(x_rdchar(codes, rdlen, fw, row)); e.type = 2; row++; }
		else { e.chr = (uint8_t)x_dna(refc); e.qchr = '-'; e.type = 1; }
	}
	a->nedits = (int16_t)n;
	u.arenaTop = ((uint32_t)off << 3) + (((uint32_t)(sizeof(XAln) + (size_t)n * sizeof(XEdit)) + 7u) & ~7u);
	return off;
}
// exact / 1-mismatch end-to-end hit at a resolved offset (SwDriver::extendSeeds eeMode, aligner_sw_driver.cpp:1172-1186)
XE_HD inline uint16_t x_aln_from_ee(XUnit &u, const XEEHit &h, int64_t tidx, int64_t refoff, bool fw, int rdlen) {
	const uint16_t off = x_new_aln(u, h.hasEdit ? 1 : 0);
	if(off == 0xffff) return off;
	XAln *a = x_aln(u, off);
	a->tidx = (int32_t)tidx; a->refoff = refoff; a->fw = fw; a->score = h.score; a->rdlen = (int16_t)rdlen; a->ns = (uint8_t)h.ns(); a->refns = (uint8_t)h.refns();
	if(h.hasEdit) { XEdit &e = a->edits()[0]; e.pos = (int16_t)(fw ? h.pos : rdlen - h.pos - 1); e.chr = h.chr; e.qchr = h.qchr; e.type = 3; e.pad = 0; }
	return off;
}

// alignment -> device op string (policy_engine.py: aln_to_ops); returns nops (clamped writes)
XE_HD inline int x_aln_to_ops(const XAln *a, const uint8_t *codes, uint8_t *ops, uint32_t maxOps) {
	const XEdit *ed = a->edits();
	const int row0 = a->trimLeft(), ext = a->ext(), rdlen = a->rdlen;
	// count first (ops are stored last column first)
	int n = ext;
	for(int k = 0; k < a->nedits; k++) n += ed[k].type == 1;
	int k = 0, w = 0;
	for(int rel = 0; rel < ext; rel++) {
		while(k < a->nedits && ed[k].pos == rel && ed[k].type == 1) { const int idx = n - 1 - w; if(idx >= 0 && (uint32_t)idx < maxOps) ops[idx] = (uint8_t)(BT2G_OP_READGAP | (x_code(ed[k].chr) << 2)); w++; k++; }
		uint8_t op;
		if(k < a->nedits && ed[k].pos == rel) { op = ed[k].type == 2 ? (uint8_t)BT2G_OP_REFGAP : (uint8_t)(BT2G_OP_MM | (x_code(ed[k].chr) << 2)); k++; }
		else op = (uint8_t)(BT2G_OP_MATCH | (x_rdchar(codes, rdlen, a->fw != 0, row0 + rel) << 2));
		const int idx = n - 1 - w; if(idx >= 0 && (uint32_t)idx < maxOps) ops[idx] = op; w++;
	}
	return n;
}

// ---------------------------------------------------------------------------------------------- sinks
XE_HD inline bool x_ps_done_with_mate(const XUnit &u, bool mate1) {
	const int m = mate1 ? 0 : 1;
	if(!u.doneUnp[m] || !u.doneConcord) return false;
	if(!u.doneDiscord && u.nunp[m] == 0) return false;
	return true;
}
XE_HD inline void x_ps_update_done(XUnit &u) { u.psDone = u.doneUnp[0] && u.doneUnp[1] && u.doneDiscord && u.doneConcord; }
// ReportingState::foundConcordant / foundUnpaired (aln_sink.cpp:95-300), as PairedSink::report of policy_engine.cpp
XE_HD inline bool x_ps_report(XUnit &u, const XParams &P, int a1, int a2) {      // arena offsets or -1
	if(a1 >= 0 && a2 >= 0) {
		u.nconcord++;
		if(!P.mmode && u.nconcord >= u.khits) u.doneConcord = u.exitConcordK = 1;
		else if(P.mmode && u.nconcord > u.mhits) u.doneConcord = u.exitConcordM = 1;
		u.doneDiscord = 1;
		if(u.doneConcord && !u.exitConcordM) u.doneUnp[0] = u.doneUnp[1] = 1;
		x_ps_update_done(u);
		if(u.nrs12 >= XE_LIST) { XE_FB(u); return true; }
		u.rs1[u.nrs12] = (uint16_t)a1; u.rs2[u.nrs12] = (uint16_t)a2; u.nrs12++;
		const int64_t sc = (int64_t)x_aln(u, (uint16_t)a1)->score + x_aln(u, (uint16_t)a2)->score;
		if(sc > u.bestPair) { u.best2Pair = u.bestPair; u.bestPair = sc; } else if(sc > u.best2Pair) u.best2Pair = sc;
	} else {
		const int m = a1 >= 0 ? 0 : 1;
		const int a = a1 >= 0 ? a1 : a2;
		u.nunp[m]++;
		if(!u.doneUnp[m]) {
			if(!P.mmode && u.nunp[m] >= u.khits) { u.doneUnp[m] = 1; x_ps_update_done(u); }
			else if(P.mmode && u.nunp[m] > u.mhits) { u.doneUnp[m] = 1; x_ps_update_done(u); }
		}
		if(u.nunp[m] > 1) u.doneDiscord = 1;
		uint16_t &cnt = m == 0 ? u.nrs1u : u.nrs2u;
		if(cnt >= XE_LIST) { XE_FB(u); return true; }
		(m == 0 ? u.rs1u : u.rs2u)[cnt++] = (uint16_t)a;
	}
	return u.psDone != 0;
}
XE_HD inline bool x_us_report(XUnit &u, const XParams &P, uint16_t a) {
	if(u.nus >= XE_LIST) { XE_FB(u); return true; }
	u.usAlns[u.nus++] = a;
	if(!u.usDone) {
		if(!P.mmode && (int64_t)u.nus >= u.khits) u.usDone = u.usExitK = 1;
		else if(P.mmode && (int64_t)u.nus > u.mhits) u.usDone = u.usExitM = 1;
	}
	const int64_t sc = x_aln(u, a)->score;
	if(sc > u.usBest) { u.usBest2 = u.usBest; u.usBest = sc; } else if(sc > u.usBest2) u.usBest2 = sc;
	return u.usDone != 0;
}

XE_HD inline int64_t x_tightened(const XUnit &u, int64_t bestPairScore) {
	int64_t ps = u.best2Pair + ((u.bestPair - u.best2Pair) * 3) / 4;     // tighten == 3
	if(ps < bestPairScore) ps++;
	return ps;
}

// ---------------------------------------------------------------------------------------------- the engine
// Svc supplies the read batch, the answers of the batched requests and the inline primitives:
//   const uint8_t *codes(int read), *quals(int read); int rdlen(int read); uint32_t randSeed(int read)
//   void sweep(int read, int mined[2], uint64_t tb[4])                                   (exactSweep, computed at admission)
//   int mmCount(int slot, int task); const bt2g_mm_hit *mmHits(int slot, int task); int mmMax()   (answer of XR_ONE_MM)
//   int nSeeds(int read); const uint64_t *seedRange(int read, int strand, int i)         (answer of XR_SEED: topf,botf,topb,botb)
//   const bt2g_dp_summary *dpSumm(int slot, bool mate); const bt2g_dp_cand *dpCands(..); const bt2g_dp_aln *dpAlns(..);
//   const uint8_t *dpOps(int slot, bool mate, int k); int dpMaxAlns()                   (answer of XR_DP / XR_DP_MATE)
//   bool resolve(uint64_t row, int qlen, bool reject, int64_t &tidx, int64_t &toff, int64_t &tlen)
//   void extend(int read, bool fw, int rdoff, int seedlen, const uint64_t rng[4], int &nlex, int &nrex)
//   int ungapped(int read, bool fw, int64_t tidx, int64_t refoff, int64_t tlen, int64_t minsc, bt2g_ungapped_result &r)
//   int refChar(int64_t tidx, int64_t off)
//   static constexpr bool kReport: finishRead / finishPair leave the sink lists in report order for x_report_entry (-k / -a);
//   false compiles the -M-only state machine
template <typename Svc>
struct XEngine {
	const XParams &P; XUnit &u; Svc &svc;
	XE_HD XEngine(const XParams &p, XUnit &unit, Svc &s) : P(p), u(unit), svc(s) {}

	XE_HD int64_t mapq(int64_t best, bool hasSec, int64_t sec, int64_t scMin, int64_t perfect) const {
		if(!P.mmode && !hasSec) return 255;
		return mapq_v2(best, hasSec, sec, scMin, perfect, !P.local);
	}

	// ---- SeedResults views over the seed-search answer
	XE_HD int64_t shSize(const XMate &c, bool fw, int i) const { const uint64_t *h = svc.seedRange(c.idx, fw ? 0 : 1, i); return h[1] > h[0] ? (int64_t)(h[1] - h[0]) : 0; }
	XE_HD void fillSeedHits(XMate &c, int interval, int offset, int seedlen) {
		c.shN = svc.nSeeds(c.idx); c.shInterval = interval; c.shOffset = offset; c.shSeedlen = seedlen; c.shNonz = 0; c.shNelt = 0;
		if(c.shN > XE_MAX_SEEDS) { XE_FB(u); c.shN = XE_MAX_SEEDS; }
		for(int f = 0; f < 2; f++) for(int i = 0; i < c.shN; i++) { const int64_t sz = shSize(c, f == 0, i); if(sz > 0) { c.shNonz++; c.shNelt += sz; } }
	}
	XE_HD void rankSeedHits(XMate &c) {                        // SeedResults::rankSeedHits (aligner_seed.h:1019-1080)
		const int num = c.shN;
		c.nranks = 0;
		if(P.all) {
			for(int i = 1; i < num; i++) for(int f = 0; f < 2; f++) if(shSize(c, f == 0, i) > 0) c.ranks[c.nranks++] = (uint8_t)(i | (f == 0 ? 0x80 : 0));
			if(num && shSize(c, true, 0) > 0) c.ranks[c.nranks++] = 0x80;
			if(num && shSize(c, false, 0) > 0) c.ranks[c.nranks++] = 0;
			return;
		}
		uint64_t sfw = 0, src = 0;                             // sorted flags per offset index (num <= 64)
		// range sizes once (thread-local), capped like the comparison below: the selection scans them nonz x 2 x num times
		uint32_t szs[2][XE_MAX_SEEDS];
		for(int f = 0; f < 2; f++) for(int i = 0; i < num; i++) { const int64_t z = shSize(c, f == 0, i); szs[f][i] = z > 0xffffffffll ? 0xffffffffu : (uint32_t)z; }
		while((int64_t)c.nranks < c.shNonz) {
			uint32_t minsz = 0xffffffffu; int minidx = 0; bool minfw = true;
			const int rb = u.rnd.boolean();
			for(int fwi = 0; fwi < 2; fwi++) {
				const bool fw = fwi == (rb ? 1 : 0);
				const uint64_t srt = fw ? sfw : src;
				const uint32_t *sz = szs[fw ? 0 : 1];
				int i = (int)(u.rnd.u32() % (uint32_t)num);
				if(minsz == 1u) continue;                       // (nothing is smaller than a range of one row; the draw above is still made)
				for(int t = 0; t < num; t++) {
					if(sz[i] > 0 && !((srt >> i) & 1) && sz[i] < minsz) { minsz = sz[i]; minidx = i; minfw = fw; if(minsz == 1u) break; }
					if(++i == num) i = 0;
				}
			}
			if(minfw) sfw |= (uint64_t)1 << minidx; else src |= (uint64_t)1 << minidx;
			c.ranks[c.nranks++] = (uint8_t)(minidx | (minfw ? 0x80 : 0));
		}
	}

	// ---- eeSaTups (aligner_sw_driver.cpp:66-290)
	XE_HD void addEnt(uint64_t topf, int64_t size, int rdoff, int seedlen, bool fw, int ee, bool needRand) {
		if(u.nents >= XE_ENTS) { XE_FB(u); return; }
		XEnt &e = u.ents[u.nents++];
		e.topf = topf; e.size = (int32_t)size; e.rdoff = (int16_t)rdoff; e.seedlen = (int16_t)seedlen; e.fw = fw; e.ee = (int8_t)ee; e.done1 = 0; e.mateStreak = 0;
		e.rix = 0xff;
		if(needRand && size > 1) { e.rix = (uint8_t)x_new_rand(u, (uint64_t)size, P.all != 0); if(XE_RANDS > 255 || e.rix == 0xff) XE_FB(u); }
	}
	XE_HD void eeAdd(int hi, int64_t &nelt, int64_t maxelt, bool &done) {
		const XEEHit &hit = u.hitl[hi];
		uint64_t tops[2] = {hit.top, 0}, bots[2] = {hit.bot, 0};
		const int64_t width = (int64_t)(hit.bot - hit.top);
		if(width <= 0) return;
		if(nelt + width > maxelt) {
			const int64_t trim = (nelt + width) - maxelt;
			const uint64_t rn = (P.offSize == 4 ? (uint64_t)u.rnd.u32() : u.rnd.u64()) % (uint64_t)width;
			const int64_t newwidth = width - trim;
			if(hit.top + rn + newwidth > hit.bot) { tops[0] = hit.top + rn; bots[0] = hit.bot; tops[1] = hit.top; bots[1] = hit.top + newwidth - (bots[0] - tops[0]); }
			else { tops[0] = hit.top + rn; bots[0] = tops[0] + newwidth; }
		}
		const XMate &c = u.m[u.cur];
		for(int i = 0; i < 2; i++) {
			if(done || bots[i] <= tops[i]) break;
			const int64_t w = (int64_t)(bots[i] - tops[i]);
			addEnt(tops[i], w, 0, c.rdlen, hit.fw != 0, hi, true);
			nelt += w;
			if(nelt >= maxelt) done = true;
		}
	}
	XE_HD void resetEnts() { u.nents = 0; u.nrands = 0; u.nseenPool = 0; u.nhitl = 0; }
	// useEe: take the mate's exact end-to-end hits (c.ee); the mate's 1-mismatch hits (c.mm1) always follow
	XE_HD void eeSaTups(bool useEe) {
		XMate &c = u.m[u.cur];
		resetEnts();
		int64_t nelt = 0; bool done = false;
		int64_t tot = 0, fwsz = 0;
		const int nee = useEe ? c.nee : 0;
		for(int i = 0; i < nee; i++) { const int64_t w = (int64_t)(c.ee[i].bot - c.ee[i].top); tot += w; if(c.ee[i].fw) fwsz += w; }
		if(tot > 0) {
			const uint64_t rn = (P.offSize == 4 ? (uint64_t)u.rnd.u32() : u.rnd.u64()) % (uint64_t)tot;
			const bool fwFirst = !((int64_t)rn >= fwsz);
			for(int fwi = 0; fwi < 2 && !done; fwi++) {
				const bool fw = (fwi == 0) == fwFirst;
				for(int i = 0; i < nee; i++) if((c.ee[i].fw != 0) == fw) { u.hitl[u.nhitl] = c.ee[i]; eeAdd(u.nhitl++, nelt, P.maxIters, done); break; }
			}
		}
		if(!done && c.nmm1 > 0) {
			// stable sort by score, descending; then shuffle equal-score streaks (EList::shufflePortion)
			for(int i = 1; i < c.nmm1; i++) { const XEEHit t = c.mm1[i]; int j = i - 1; while(j >= 0 && c.mm1[j].score < t.score) { c.mm1[j + 1] = c.mm1[j]; j--; } c.mm1[j + 1] = t; }
			{
				int streak = 0;
				for(int i = 1; i < c.nmm1; i++) {
					if(c.mm1[i].score == c.mm1[i - 1].score) { if(streak == 0) streak = 1; streak++; }
					else { if(streak > 1) x_shuffle_portion(c.mm1, i - streak, streak, u.rnd); streak = 0; }
				}
				if(streak > 1) x_shuffle_portion(c.mm1, c.nmm1 - streak, streak, u.rnd);
			}
			for(int i = 0; i < c.nmm1; i++) { if(done) break; u.hitl[u.nhitl] = c.mm1[i]; eeAdd(u.nhitl++, nelt, P.maxIters, done); }
		}
	}

	// ---- prioritizeSATupsRands (aligner_sw_driver.cpp:490-725) with SwDriver::extend inline
	XE_HD int64_t prioritize() {
		XMate &c = u.m[u.cur];
		resetEnts();
		u.nsats = 0;
		int64_t nelt = 0;
		for(int ri = 0; ri < c.nranks; ri++) {
			const int offidx = c.ranks[ri] & 0x7f; const bool fw = (c.ranks[ri] & 0x80) != 0;
			const uint64_t *h = svc.seedRange(c.idx, fw ? 0 : 1, offidx);
			const int64_t sz = (int64_t)(h[1] - h[0]);
			const int rdoff = c.shOffset + offidx * c.shInterval, seedlen = c.shSeedlen;
			nelt += sz;
			const int st = fw ? 0 : 1;
			bool skip = false;
			for(int x = 0; x < c.nexr[st]; x++) { const XExr &e = c.exr[st][x]; if(e.p5 <= rdoff && e.p5 + e.len >= rdoff + seedlen && sz <= e.size) { skip = true; break; } }
			if(skip) { nelt -= sz; continue; }
			if(u.nsats >= XE_SATS) { XE_FB(u); break; }
			XSat &sp = u.sats[u.nsats++];
			sp.topf = h[0]; sp.topb = h[2]; sp.size = sz; sp.fw = fw; sp.offidx = (uint8_t)offidx; sp.rdoff = (int16_t)rdoff; sp.seedlen = (int16_t)seedlen;
			sp.rix = 0xff; sp.elim = 0; sp.mass = 0.0;
			int nlex = 0, nrex = 0;
			svc.extend(c.idx, fw, rdoff, seedlen, h, nlex, nrex);
			sp.nlex = (uint8_t)nlex; sp.nrex = (uint8_t)nrex;
			if(nlex > 0 || nrex > 0) {
				if(c.nexr[st] >= XE_EXR) { XE_FB(u); }
				else { XExr &e = c.exr[st][c.nexr[st]++]; e.p5 = rdoff - (fw ? nlex : nrex); e.len = seedlen + nlex + nrex; e.size = sz; }
			}
		}
		const int ns = u.nsats;
		int nsmall = 0;
		for(int i = 0; i < ns; i++) nsmall += u.sats[i].size <= 5;
		// SATupleAndPos::operator< : size, topf, offidx, rdoff, seedlen, fw first
		for(int i = 1; i < ns; i++) {
			const XSat t = u.sats[i]; int j = i - 1;
			while(j >= 0) {
				const XSat &b = u.sats[j];
				bool less;                                       // t < b ?
				if(t.size != b.size) less = t.size < b.size;
				else if(t.topf != b.topf) less = t.topf < b.topf;
				else if(t.offidx != b.offidx) less = t.offidx < b.offidx;
				else if(t.rdoff != b.rdoff) less = t.rdoff < b.rdoff;
				else if(t.seedlen != b.seedlen) less = t.seedlen < b.seedlen;
				else less = t.fw && !b.fw;
				if(!less) break;
				u.sats[j + 1] = u.sats[j]; j--;
			}
			u.sats[j + 1] = t;
		}
		int64_t added = 0;
		int j = 0;
		while(j < nsmall && added < P.maxIters) {
			const XSat &s = u.sats[j];
			addEnt(s.topf, s.size, s.rdoff, s.seedlen, s.fw != 0, -1, true);
			added += s.size; j++;
		}
		if(added >= P.maxIters || nsmall == ns) return added;
		// RowSampler (aligner_sw_driver.h:179-256)
		const int nl = ns - nsmall;
		double mass = 0.0;
		for(int i = 0; i < nl; i++) {
			XSat &s = u.sats[nsmall + i];
			double num = (double)(s.nlex + s.nrex + 1); num *= num;
			double den = (double)s.size; den *= den;
			s.mass = num / den; mass += s.mass; s.elim = 0;
		}
		while(added < P.maxIters && added < nelt) {
			const double rd = u.rnd.flt() * mass;
			double sofar = 0.0; int pick = 0, last = 0;
			bool got = false;
			for(int i = 0; i < nl; i++) if(!u.sats[nsmall + i].elim) { last = i; sofar += u.sats[nsmall + i].mass; if(rd < sofar) { pick = i; got = true; break; } }
			if(!got) pick = last;
			XSat &s = u.sats[nsmall + pick];
			if(s.rix == 0xff) { s.rix = (uint8_t)x_new_rand(u, (uint64_t)s.size, P.all != 0); }
			if(u.fallback) break;
			const uint32_t r = x_rand_next(u, s.rix, u.rnd);
			if(x_rand_done(u.rands[s.rix])) { s.elim = 1; mass -= s.mass; }
			addEnt(s.topf + r, 1, s.rdoff, s.seedlen, s.fw != 0, -1, false);
			added++;
			if(u.fallback) break;
		}
		return added;
	}
	XE_HD bool entDone(const XEnt &e) const { return e.rix == 0xff ? e.done1 != 0 : x_rand_done(u.rands[e.rix]); }
	XE_HD uint32_t entNext(XEnt &e) { if(e.rix == 0xff) { e.done1 = 1; return 0; } return x_rand_next(u, e.rix, u.rnd); }
	XE_HD void entSetDone(XEnt &e) { if(e.rix == 0xff) e.done1 = 1; else u.rands[e.rix].cur = u.rands[e.rix].n; }

	XE_HD bool dpU8(int64_t best, int64_t minsc, const XMate &mt) const {
		if(!P.local) return minsc >= -254;
		int bias = P.nPen;
		const uint8_t *q = svc.quals(mt.idx);
		for(int i = 0; i < mt.rdlen; i++) { const int p = P.mmPenalty((int)q[i] - 33); if(p > bias) bias = p; }
		return best + bias < 255;
	}
	XE_HD void reseed(bool u8) { const uint32_t rs = u.rnd.u32() + 1u; u.rnd.init(u8 ? rs + 1u : rs); }

	// copy the anchor DP's attempt list into the unit (its buffers are reused by the next wave)
	XE_HD bool loadAnchorDp(const XMate &c) {
		const bt2g_dp_summary *s = svc.dpSumm(u.dpSlot, false);
		u.natt = 0; u.attCursor = 0;
		if(s->flags) { XE_FB(u); return false; }
		if(!s->found) return false;
		const bt2g_dp_cand *cands = svc.dpCands(u.dpSlot, false);
		const bt2g_dp_aln *alns = svc.dpAlns(u.dpSlot, false);
		int k = 0;
		for(int ci = 0; ci < s->ncand; ci++) {
			const int f = cands[ci].fate;
			if(f != BT2G_CAND_SUCCEEDED && f != BT2G_CAND_FAILED) continue;
			if(u.natt >= XE_ATT) { XE_FB(u); return false; }
			u.attScore[u.natt] = (int16_t)cands[ci].score;
			uint16_t ao = 0xffff;
			if(f == BT2G_CAND_SUCCEEDED) {
				if(k >= svc.dpMaxAlns()) { XE_FB(u); return false; }
				ao = x_aln_from_dp(u, u.rqProb, alns[k], svc.dpOps(u.dpSlot, false, k), svc.codes(c.idx), c.rdlen);
				if(ao == 0xffff) return false;
				k++;
			}
			u.attAln[u.natt++] = ao;
		}
		u.dpU8 = dpU8(s->best, c.minsc, c);
		return true;
	}
	// SwAligner::nextAlignment over the anchor DP's attempts: candidates below minsc are skipped, every attempt reseeds the RNG
	XE_HD bool nextAnchorAln(int64_t minsc, uint16_t &out) {
		while(u.attCursor < u.natt) {
			const int i = u.attCursor++;
			if(u.attScore[i] < minsc) continue;
			reseed(u.dpU8 != 0);
			if(u.attAln[i] != 0xffff) { out = u.attAln[i]; return true; }
		}
		return false;
	}
	// the same over the mate DP's answer, read in place (it is consumed within one step)
	XE_HD bool nextMateAln(const XMate &o, int64_t minsc, uint16_t &out) {
		const bt2g_dp_summary *s = svc.dpSumm(u.dpSlot, true);
		const bt2g_dp_cand *cands = svc.dpCands(u.dpSlot, true);
		const bt2g_dp_aln *alns = svc.dpAlns(u.dpSlot, true);
		while(u.mateCursor < s->ncand) {
			const int ci = u.mateCursor++;
			const int f = cands[ci].fate;
			if(f != BT2G_CAND_SUCCEEDED && f != BT2G_CAND_FAILED) continue;
			const bool ok = f == BT2G_CAND_SUCCEEDED;
			const int k = u.mateAlnK;
			if(ok) u.mateAlnK++;
			if(cands[ci].score < minsc) continue;
			reseed(u.odpU8 != 0);
			if(ok) {
				if(k >= svc.dpMaxAlns()) { XE_FB(u); return false; }
				out = x_aln_from_dp(u, u.rqProb, alns[k], svc.dpOps(u.dpSlot, true, k), svc.codes(o.idx), o.rdlen);
				return out != 0xffff;
			}
		}
		return false;
	}

	XE_HD void setDpReq(const XMate &c, bool fw, int64_t tidx, const XRect &rect, int64_t minsc, int rdlen) {
		bt2g_dp_problem &p = u.rqProb;
		p.read_idx = (uint32_t)c.idx; p.fw = fw ? 1u : 0u; p.tidx = (uint64_t)tidx; p.refl = rect.refl; p.refr = rect.refr;
		p.triml = (int32_t)rect.triml; p.corel = (int32_t)rect.corel; p.corer = (int32_t)rect.corer;
		p.minsc = (int32_t)minsc; p.nceil = P.nCeilRaw(rdlen); p.reserved = 0;
	}

	// ungapped alignment (SwAligner::ungappedAlign through Svc) -> arena record; returns the status
	XE_HD int ungapped(const XMate &c, bool fw, int64_t tidx, int64_t refoff, int64_t tlen, uint16_t &out) {
		bt2g_ungapped_result r;
		const int st = svc.ungapped(c.idx, fw, tidx, refoff, tlen, c.minsc, r);
		if(st != 1) return st;
		const uint8_t *cd = svc.codes(c.idx);
		const int len = c.rdlen, rowi = r.rowi, rowf = r.rowf;
		int ned = 0;
		for(int i = rowi; i <= rowf; i++) { const int f = svc.refChar(tidx, refoff + i); if(f > 3 || x_rdchar(cd, len, fw, i) != f) ned++; }
		out = x_new_aln(u, ned);
		if(out == 0xffff) return st;
		XAln *a = x_aln(u, out);
		XEdit *ed = a->edits();
		int n = 0;
		for(int i = rowi; i <= rowf; i++) {
			const int f = svc.refChar(tidx, refoff + i), rc = x_rdchar(cd, len, fw, i);
			if(f > 3 || rc != f) { XEdit &e = ed[n++]; e.pos = (int16_t)(i - rowi); e.chr = (uint8_t)x_dna(f); e.qchr = (uint8_t)x_dna(rc); e.type = 3; e.pad = 0; }
		}
		const int tl = rowi, tr = len - 1 - rowf;
		a->tidx = (int32_t)tidx; a->refoff = refoff + rowi; a->fw = fw; a->score = r.score; a->rdlen = (int16_t)len; a->ns = (uint8_t)r.ns; a->refns = (uint8_t)r.refns;
		a->trim5 = (int16_t)(fw ? tl : tr); a->trim3 = (int16_t)(fw ? tr : tl);
		return st;
	}

	XE_HD void tightenUnpaired(XMate &c) {
		if(!(P.mmode && u.usBest2 != XE_MIN_I64)) return;
		const int64_t bot = u.usBest2 + ((u.usBest - u.usBest2) * 3) / 4;      // tighten == 3
		if(bot >= c.minsc) { c.minsc = bot; if(c.minsc < c.perfect) c.minsc++; }
	}

	XE_HD int stepExtPaired();
	XE_HD int stepExtUnpaired();
	XE_HD int stepPair();
	XE_HD int stepRead();
	XE_HD void finishPair();
	XE_HD void finishRead();
	XE_HD void loadMm1(XMate &c, int64_t *neltOut);
};

// protothread plumbing: resume at the saved program counter; a request returns to the caller and re-enters right after it
#define XE_WAIT(PCVAR, N, REQ) do { PCVAR = N; return (REQ); case N:; } while(0)

// 1-mismatch hits of the answered XR_ONE_MM request -> c.mm1 (task order: (fw, fw index), (fw, mirror), (rc, fw), (rc, mirror))
template <typename Svc>
XE_HD void XEngine<Svc>::loadMm1(XMate &c, int64_t *neltOut) {
	c.nmm1 = 0;
	for(int task = 0; task < 4; task++) {
		const int n = svc.mmCount(u.dpSlot, task);
		const bt2g_mm_hit *h = svc.mmHits(u.dpSlot, task);
		if(n > svc.mmMax()) { XE_FB(u); return; }
		for(int j = 0; j < n; j++) {
			if(c.nmm1 >= XE_MM1) { XE_FB(u); return; }
			XEEHit &e = c.mm1[c.nmm1++];
			e.top = h[j].top; e.bot = h[j].bot; e.fw = task < 2; e.score = h[j].score; e.hasEdit = 1; e.pos = (int16_t)h[j].pos;
			e.chr = (uint8_t)x_dna(h[j].chr); e.qchr = (uint8_t)x_dna(h[j].qchr); e.pad[0] = e.pad[1] = 0;
			if(neltOut) *neltOut += (int64_t)(h[j].bot - h[j].top);
		}
	}
}

// ---------------------------------------------------------------------------------------------- extendSeedsPaired
// SwDriver::extendSeedsPaired (aligner_sw_driver.cpp:1582-2637) as policy_engine.cpp restates it.  Arguments in
// u.xAi (anchor mate), u.xUseSh (seed hits of the mate), u.xUseEe (its exact end-to-end hits); result in u.xRet.
template <typename Svc>
XE_HD int XEngine<Svc>::stepExtPaired() {
	const bool anchor1 = u.xAi == 0;
	XMate &c = u.m[u.xAi], &o = u.m[u.xAi ^ 1];
	const int rdlen = c.rdlen, ordlen = o.rdlen;
	const bool oppFilt = !o.filt;
	const int64_t operfect = o.perfect, bestPairScore = c.perfect + operfect;
	const bool canTighten = P.mmode != 0;
	XRect rect;
	switch(u.pcExt) {
	case 0:
		u.cur = u.xAi;
		if(canTighten && u.best2Pair != XE_MIN_I64) { const int64_t nc = x_tightened(u, bestPairScore) - operfect; if(nc > c.minsc) c.minsc = nc; }
		u.nonz = u.xUseSh ? c.shNonz : 0;
		u.eeMode = (u.xUseEe && c.nee > 0) || c.nmm1 > 0; u.firstEe = 1; u.firstExtend = 1; u.swMateImmediately = 1;
		u.nEeFail = u.nUgFail = u.nDpFail = 0; u.neltLeft = 0;
		u.streak = u.streakCur;
		u.nents = 0;
		for(;;) {
			if(u.eeMode) { if(u.firstEe) { u.firstEe = 0; eeSaTups(u.xUseEe != 0); if(u.fallback) return XR_FALLBACK; } else u.eeMode = 0; }
			if(!u.eeMode) {
				if(u.nonz == 0) { u.xRet = EXHAUSTED; return XR_DONE; }
				if(P.mmode && c.minsc == c.perfect) { u.xRet = PERFECT; return XR_DONE; }
				if(u.firstExtend) { u.neltLeft = prioritize(); u.firstExtend = 0; if(u.fallback) return XR_FALLBACK; }
				if(u.neltLeft == 0) break;
			}
			for(u.si = 0; u.si < u.nents; u.si++) {
				if(u.eeMode && u.hitl[u.ents[u.si].ee].score < c.minsc) { u.xRet = PERFECT; return XR_DONE; }
				u.isSmall = u.ents[u.si].size < 5; u.fw = u.ents[u.si].fw;
				u.rdoff = u.ents[u.si].rdoff;
				if(!u.fw) u.rdoff = rdlen - u.rdoff - u.ents[u.si].seedlen;
				u.first = 1;
				while(!entDone(u.ents[u.si]) && (u.first || u.isSmall || u.eeMode)) {
					if(c.minsc == c.perfect) { if(!u.eeMode || u.hitl[u.ents[u.si].ee].score < c.perfect) { u.xRet = PERFECT; return XR_DONE; } }
					else if(u.eeMode && u.hitl[u.ents[u.si].ee].score < c.minsc) break;
					if(u.nDps >= P.maxDp || u.nMateDps >= P.maxDp || u.nUgs >= P.maxUg || u.nIters >= P.maxIters) { u.xRet = HARD_LIMIT; return XR_DONE; }
					if(u.eeMode && u.nEeFail >= u.streak) { u.xRet = SOFT_LIMIT; return XR_DONE; }
					if(!u.eeMode && (u.nDpFail >= u.streak || u.nUgFail >= u.streak)) { u.xRet = SOFT_LIMIT; return XR_DONE; }
					if(u.ents[u.si].mateStreak >= P.maxMateStreak) { entSetDone(u.ents[u.si]); break; }
					u.nIters++; u.first = 0;
					{
						const uint32_t elt = entNext(u.ents[u.si]);
						if(u.fallback) return XR_FALLBACK;
						u.neltLeft--;
						if(!svc.resolve(u.ents[u.si].topf + elt, u.ents[u.si].seedlen, u.eeMode != 0, u.tidx, u.toff, u.tlen)) continue;
					}
					u.refoff = u.toff - u.rdoff;
					if(x_seen_present(c, u.tidx, u.fw != 0, u.refoff)) continue;
					u.readGaps = 0; u.refGaps = 0;
					{
						bool ungappedOk = false;
						if(!u.eeMode) { u.readGaps = P.maxReadGaps(c.minsc, rdlen); u.refGaps = P.maxRefGaps(c.minsc, rdlen); ungappedOk = u.readGaps == 0 && u.refGaps == 0; }
						u.state = 0; u.fixedAln = 0xffff;
						if(u.eeMode) {
							u.fixedAln = x_aln_from_ee(u, u.hitl[u.ents[u.si].ee], u.tidx, u.refoff, u.fw != 0, rdlen); u.state = 1;
							x_seen_add(u, c, u.tidx, u.fw != 0, u.refoff, 1); u.nEeFail++;
						} else if(ungappedOk) {
							uint16_t ua = 0xffff;
							const int st = ungapped(c, u.fw != 0, u.tidx, u.refoff, u.tlen, ua);
							x_seen_add(u, c, u.tidx, u.fw != 0, u.refoff, 1);
							u.nUgs++; u.nUgFail++;
							if(st == 0) continue;
							if(st == 1) { u.fixedAln = ua; u.state = 2; }
						}
						if(u.fallback) return XR_FALLBACK;
					}
					if(u.state == 0) {
						{
							const bool found = x_frame_seed(u.refoff, rdlen, u.tlen, u.readGaps, u.refGaps, 15, rect);
							x_seen_add(u, c, u.tidx, u.fw != 0, u.refoff, 1);
							if(!found) continue;
							x_seen_add(u, c, u.tidx, u.fw != 0, rect.reflPre + rect.corel, rect.corer - rect.corel + 1);
							if(u.fallback) return XR_FALLBACK;
							setDpReq(c, u.fw != 0, u.tidx, rect, c.minsc, rdlen);
						}
						XE_WAIT(u.pcExt, 1, XR_DP);
						u.nDps++; u.nDpFail++;
						if(!loadAnchorDp(c)) { if(u.fallback) return XR_FALLBACK; continue; }
					}
					u.firstInner = 1; u.foundConcordant = 0;
					for(;;) {
						if(u.state != 0) { if(!u.firstInner) break; u.curAln = u.fixedAln; }
						else if(!nextAnchorAln(c.minsc, u.curAln)) break;
						u.firstInner = 0;
						if(x_red_overlap(u, 0, u.curAln)) continue;
						x_red_add(u, 0, u.curAln);
						if(x_ps_done_with_mate(u, !anchor1) && !x_ps_done_with_mate(u, anchor1)) u.swMateImmediately = 0;
						if(u.swMateImmediately) {
							u.foundMate = !oppFilt;
							u.ominscCur = o.minsc;
							if(u.foundMate) {
								const XAln *a = x_aln(u, u.curAln);
								if(canTighten && u.best2Pair != XE_MIN_I64) { const int64_t nc = x_tightened(u, bestPairScore) - a->score; if(nc > u.ominscCur) u.ominscCur = nc; }
								const int ordgaps = P.maxReadGaps(u.ominscCur, ordlen), orfgaps = P.maxRefGaps(u.ominscCur, ordlen);
								bool oleft = false, ofw = false; int64_t oll = 0, olr = 0, orl = 0, orr = 0;
								bool fm = pe_other_mate(P.pe, anchor1, u.fw != 0, a->refoff, (int64_t)ordlen + ordgaps, (uint64_t)(anchor1 ? rdlen : ordlen),
								                        (uint64_t)(anchor1 ? ordlen : rdlen), oleft, oll, olr, orl, orr, ofw);
								if(fm) fm = x_frame_mate(!oleft, oll, olr, orl, orr, ordlen, u.tlen, ordgaps, orfgaps, 15, rect);
								u.foundMate = fm;
								if(fm) setDpReq(o, ofw, u.tidx, rect, u.ominscCur, ordlen);
							}
							if(u.foundMate) {
								XE_WAIT(u.pcExt, 2, XR_DP_MATE);
								u.nMateDps++;
								{
									const bt2g_dp_summary *s = svc.dpSumm(u.dpSlot, true);
									if(s->flags) { XE_FB(u); return XR_FALLBACK; }
									u.foundMate = s->found != 0;
									u.mateCursor = 0; u.mateAlnK = 0;
									if(u.foundMate) u.odpU8 = dpU8(s->best, u.ominscCur, o);
								}
							}
							u.didAnchor = 0; u.brk = 0;
							for(;;) {
								uint16_t oaOff = 0xffff; u.haveOa = 0;
								if(u.foundMate) { u.haveOa = nextMateAln(o, u.ominscCur, oaOff); if(u.fallback) return XR_FALLBACK; u.foundMate = u.haveOa; }
								int64_t oext = 0;
								if(u.foundMate) {
									if(!x_red_overlap(u, 0, oaOff)) x_red_add(u, 0, oaOff);
									const XAln *oa = x_aln(u, oaOff);
									oext = oa->refExtent();
									if(oa->refoff < 0 || oa->refoff + oext > u.tlen) u.foundMate = 0;
								}
								int pairCl = 5;
								if(u.foundMate) {
									const XAln *a = x_aln(u, u.curAln), *oa = x_aln(u, oaOff);
									const int64_t aext = a->refExtent();
									const XAln *a1 = anchor1 ? a : oa, *a2 = anchor1 ? oa : a;
									pairCl = pe_classify(P.pe, a1->refoff, (uint64_t)(anchor1 ? aext : oext), a1->fw != 0, a2->refoff, (uint64_t)(anchor1 ? oext : aext), a2->fw != 0);
								}
								if(u.doneConcord) u.foundMate = 0;
								if(u.foundMate) {
									bool doneUnpaired = false;
									if(!anchor1 || !u.didAnchor) {
										if(anchor1) u.didAnchor = 1;
										const uint16_t r1 = anchor1 ? u.curAln : oaOff;
										if(!x_red_overlap(u, 1, r1)) { x_red_add(u, 1, r1); if(x_ps_report(u, P, r1, -1)) doneUnpaired = true; }
									}
									if(anchor1 || !u.didAnchor) {
										if(!anchor1) u.didAnchor = 1;
										const uint16_t r2 = anchor1 ? oaOff : u.curAln;
										if(!x_red_overlap(u, 2, r2)) { x_red_add(u, 2, r2); if(x_ps_report(u, P, -1, r2)) doneUnpaired = true; }
									}
									bool donePaired = false;
									if(pairCl != 5) {
										u.foundConcordant = 1;
										if(x_ps_report(u, P, anchor1 ? u.curAln : oaOff, anchor1 ? oaOff : u.curAln)) donePaired = true;
										else if(canTighten && u.best2Pair != XE_MIN_I64) {
											const int64_t nc = x_tightened(u, bestPairScore) - operfect;
											if(nc > c.minsc) { c.minsc = nc; if(c.minsc > x_aln(u, u.curAln)->score) u.brk = 1; }
										}
									}
									if(u.fallback) return XR_FALLBACK;
									if(u.brk) break;
									if(donePaired || doneUnpaired) { u.xRet = FULFILLED; return XR_DONE; }
									if(x_ps_done_with_mate(u, anchor1)) { u.xRet = FULFILLED; return XR_DONE; }
								} else if((P.mixed || P.discord) && !u.didAnchor) {
									u.didAnchor = 1;
									if(!u.doneUnp[anchor1 ? 0 : 1]) {
										const int set = anchor1 ? 1 : 2;
										if(!x_red_overlap(u, set, u.curAln)) { x_red_add(u, set, u.curAln); if(x_ps_report(u, P, anchor1 ? u.curAln : -1, anchor1 ? -1 : u.curAln)) { u.xRet = FULFILLED; return XR_DONE; } }
									}
									if(u.fallback) return XR_FALLBACK;
									if(x_ps_done_with_mate(u, anchor1)) { u.xRet = FULFILLED; return XR_DONE; }
								}
								if(!u.haveOa) break;
							}
						} else if(P.mixed || P.discord) {
							if(!u.doneUnp[anchor1 ? 0 : 1]) {
								const int set = anchor1 ? 1 : 2;
								if(!x_red_overlap(u, set, u.curAln)) { x_red_add(u, set, u.curAln); if(x_ps_report(u, P, anchor1 ? u.curAln : -1, anchor1 ? -1 : u.curAln)) { u.xRet = FULFILLED; return XR_DONE; } }
							}
							if(u.fallback) return XR_FALLBACK;
							if(x_ps_done_with_mate(u, anchor1)) { u.xRet = FULFILLED; return XR_DONE; }
						}
					}
					if(u.foundConcordant) { u.ents[u.si].mateStreak = 0; if(u.state == 2) u.nUgFail = 0; else if(u.state == 1) u.nEeFail = 0; else u.nDpFail = 0; }
					else u.ents[u.si].mateStreak++;
				}
			}
		}
		u.xRet = EXHAUSTED;
		return XR_DONE;
	}
	XE_FB(u);
	return XR_FALLBACK;
}

// ---------------------------------------------------------------------------------------------- extendSeeds (unpaired)
// SwDriver::extendSeeds (aligner_sw_driver.cpp:921-1494).  Arguments: u.xUseSh, u.xUseEe; result in u.xRet.
template <typename Svc>
XE_HD int XEngine<Svc>::stepExtUnpaired() {
	XMate &c = u.m[0];
	const int rdlen = c.rdlen;
	XRect rect;
	switch(u.pcExt) {
	case 0:
		u.cur = 0;
		u.nonz = u.xUseSh ? c.shNonz : 0;
		u.eeMode = (u.xUseEe && c.nee > 0) || c.nmm1 > 0; u.firstEe = 1; u.firstExtend = 1;
		u.nUgFail = u.nDpFail = 0; u.neltLeft = 0;
		u.nents = 0;
		for(;;) {
			if(u.eeMode) { if(u.firstEe) { u.firstEe = 0; eeSaTups(u.xUseEe != 0); if(u.fallback) return XR_FALLBACK; } else u.eeMode = 0; }
			if(!u.eeMode) {
				if(u.nonz == 0) { u.xRet = EXHAUSTED; return XR_DONE; }
				if(c.minsc == c.perfect) { u.xRet = PERFECT; return XR_DONE; }
				if(u.firstExtend) { u.neltLeft = prioritize(); u.firstExtend = 0; if(u.fallback) return XR_FALLBACK; }
				if(u.neltLeft == 0) break;
			}
			for(u.si = 0; u.si < u.nents; u.si++) {
				if(u.eeMode && u.hitl[u.ents[u.si].ee].score < c.minsc) { u.xRet = PERFECT; return XR_DONE; }
				u.isSmall = u.ents[u.si].size < 5; u.fw = u.ents[u.si].fw;
				u.rdoff = u.ents[u.si].rdoff;
				if(!u.fw) u.rdoff = rdlen - u.rdoff - u.ents[u.si].seedlen;
				u.first = 1;
				while(!entDone(u.ents[u.si]) && (u.first || u.isSmall || u.eeMode)) {
					if(c.minsc == c.perfect) { if(!u.eeMode || u.hitl[u.ents[u.si].ee].score < c.perfect) { u.xRet = PERFECT; return XR_DONE; } }
					else if(u.eeMode && u.hitl[u.ents[u.si].ee].score < c.minsc) break;
					if(u.nDps >= P.maxDp || u.nUgs >= P.maxUg || u.nIters >= P.maxIters) { u.xRet = HARD_LIMIT; return XR_DONE; }
					u.nIters++; u.first = 0;
					{
						const uint32_t elt = entNext(u.ents[u.si]);
						if(u.fallback) return XR_FALLBACK;
						const bool ok = svc.resolve(u.ents[u.si].topf + elt, u.ents[u.si].seedlen, u.eeMode != 0, u.tidx, u.toff, u.tlen);
						if(!u.eeMode) u.neltLeft--;
						if(!ok) continue;
					}
					u.refoff = u.toff - u.rdoff;
					if(x_seen_present(c, u.tidx, u.fw != 0, u.refoff)) continue;
					u.readGaps = 0; u.refGaps = 0;
					{
						bool ungappedOk = false;
						if(!u.eeMode) { u.readGaps = P.maxReadGaps(c.minsc, rdlen); u.refGaps = P.maxRefGaps(c.minsc, rdlen); ungappedOk = u.readGaps == 0 && u.refGaps == 0; }
						u.state = 0; u.fixedAln = 0xffff;
						if(u.eeMode) {
							u.fixedAln = x_aln_from_ee(u, u.hitl[u.ents[u.si].ee], u.tidx, u.refoff, u.fw != 0, rdlen); u.state = 1;
							x_seen_add(u, c, u.tidx, u.fw != 0, u.refoff, 1);
						} else if(ungappedOk) {
							uint16_t ua = 0xffff;
							const int st = ungapped(c, u.fw != 0, u.tidx, u.refoff, u.tlen, ua);
							x_seen_add(u, c, u.tidx, u.fw != 0, u.refoff, 1);
							u.nUgs++;
							if(st == 0) { if(++u.nUgFail >= P.streak) { u.xRet = SOFT_LIMIT; return XR_DONE; } continue; }
							else if(st == -1) { if(++u.nUgFail >= P.streak) { u.xRet = SOFT_LIMIT; return XR_DONE; } }
							else { u.nUgFail = 0; u.fixedAln = ua; u.state = 2; }
						}
						if(u.fallback) return XR_FALLBACK;
					}
					if(u.state == 0) {
						{
							const bool found = x_frame_seed(u.refoff, rdlen, u.tlen, u.readGaps, u.refGaps, 15, rect);
							x_seen_add(u, c, u.tidx, u.fw != 0, u.refoff, 1);
							if(!found) continue;
							x_seen_add(u, c, u.tidx, u.fw != 0, rect.reflPre + rect.corel, rect.corer - rect.corel + 1);
							if(u.fallback) return XR_FALLBACK;
							setDpReq(c, u.fw != 0, u.tidx, rect, c.minsc, rdlen);
						}
						XE_WAIT(u.pcExt, 1, XR_DP);
						u.nDps++;
						if(!loadAnchorDp(c)) {
							if(u.fallback) return XR_FALLBACK;
							if(++u.nDpFail >= P.streak) { u.xRet = SOFT_LIMIT; return XR_DONE; }
							continue;
						}
						u.nDpFail = 0;
					}
					u.firstInner = 1;
					for(;;) {
						if(u.state != 0) { if(!u.firstInner) break; u.curAln = u.fixedAln; }
						else if(!nextAnchorAln(c.minsc, u.curAln)) break;
						u.firstInner = 0;
						if(x_red_overlap(u, 0, u.curAln)) continue;
						x_red_add(u, 0, u.curAln);
						if(x_us_report(u, P, u.curAln)) { if(u.fallback) return XR_FALLBACK; u.xRet = FULFILLED; return XR_DONE; }
						tightenUnpaired(c);
						if(u.fallback) return XR_FALLBACK;
					}
				}
			}
		}
		u.xRet = EXHAUSTED;
		return XR_DONE;
	}
	XE_FB(u);
	return XR_FALLBACK;
}

// call a sub-protothread: forwards its requests to our caller, continues here when it finishes
#define XE_CALL_EXT(N, FN) do { u.pcExt = 0; case N: { const int r_ = FN(); if(r_ != XR_DONE) { u.pc = N; return r_; } } } while(0)

// ---------------------------------------------------------------------------------------------- pairs
// multiseedSearchWorker for a pair (bt2_search.cpp:3253-4199) as policy_engine.cpp: Engine::pairSteps
template <typename Svc>
XE_HD int XEngine<Svc>::stepPair() {
	switch(u.pc) {
	case 0: {
		{
		const int i1 = (int)(2 * u.id), ls[2] = {svc.rdlen(i1), svc.rdlen(i1 + 1)};
		for(int k = 0; k < 2; k++) {
			XMate &c = u.m[k];
			c.idx = i1 + k; c.rdlen = ls[k];
			if(ls[k] > P.maxLen) { XE_FB(u); return XR_FALLBACK; }
			c.minsc = ls[k] ? P.minScore(ls[k]) : 0; c.perfect = P.perfect(ls[k]); c.nceil = ls[k] ? P.nCeil(ls[k]) : 0;
			const uint8_t *cd = svc.codes(c.idx);
			int nn = 0; for(int i = 0; i < ls[k]; i++) nn += cd[i] > 3;
			c.filt = !(ls[k] < 2 || nn > P.nCeil(ls[k]) || P.perfect(ls[k]) < P.minScore(ls[k]));
			c.nee = c.nmm1 = c.hasSh = 0; c.nexr[0] = c.nexr[1] = 0; c.nseen = 0; c.nranks = 0; c.shN = 0; c.shNonz = c.shNelt = 0;
		}
		u.both = u.m[0].filt && u.m[1].filt;
		{
			const uint32_t s1 = svc.randSeed(i1), s2 = svc.randSeed(i1 + 1);
			u.rnd.init(u.both ? (s1 ^ s2) : s1);
		}
		for(int k = 0; k < 2; k++) u.interval[k] = ls[k] ? P.seedInterval(ls[k], u.both != 0) : 1;
		int64_t streak = P.streak; u.nroundsAll = P.seedRounds;
		if(u.both) { streak = (streak + 1) / 2; u.nroundsAll = (u.nroundsAll + 1) / 2; }
		u.streakCur = streak;
		u.khits = P.khits; u.mhits = P.mhits;
		u.doneConcord = 0; u.exitConcordM = u.exitConcordK = 0; u.psDone = 0;
		u.nconcord = 0; u.nunp[0] = u.nunp[1] = 0; u.bestPair = u.best2Pair = XE_MIN_I64; u.nrs12 = u.nrs1u = u.nrs2u = 0;
		u.doneDiscord = !P.discord; u.doneUnp[0] = u.doneUnp[1] = !P.mixed;
		u.nred[0] = u.nred[1] = u.nred[2] = 0;
		u.nIters = u.nDps = u.nUgs = u.nMateDps = 0;
		const bool m1fw = P.pe.pol == 1 || P.pe.pol == 3, m2fw = P.pe.pol == 1 || P.pe.pol == 4;
		u.nofwM[0] = m1fw ? P.nofw : P.norc; u.nofwM[1] = m2fw ? P.nofw : P.norc;
		u.norcM[0] = m1fw ? P.norc : P.nofw; u.norcM[1] = m2fw ? P.norc : P.nofw;
		u.done[0] = !u.m[0].filt; u.done[1] = !u.m[1].filt;
		u.matemap[0] = 0; u.matemap[1] = 1; u.nelt[0] = u.nelt[1] = 0;
		u.mined[0][0] = u.mined[0][1] = u.mined[1][0] = u.mined[1][1] = 0;
		// ---- exact end-to-end (exactSweep answers are available from admission)
		for(int mi = 0; mi < 2; mi++) {
			const int mate = u.matemap[mi]; XMate &c = u.m[mate];
			if(!c.filt || u.done[mate] || x_ps_done_with_mate(u, mate == 0)) continue;
			uint64_t tb[4]; int mined[2];
			svc.sweep(c.idx, mined, tb);
			if(u.nofwM[mate]) { tb[0] = tb[1] = 0; mined[0] = 0; }       // (a skipped strand reports nothing)
			if(u.norcM[mate]) { tb[2] = tb[3] = 0; mined[1] = 0; }
			u.nelt[mate] = (int64_t)((tb[1] > tb[0] ? tb[1] - tb[0] : 0) + (tb[3] > tb[2] ? tb[3] - tb[2] : 0));
			u.mined[mate][0] = mined[0]; u.mined[mate][1] = mined[1];
			c.nee = 0;
			if(tb[1] > tb[0]) { XEEHit &e = c.ee[c.nee++]; e.top = tb[0]; e.bot = tb[1]; e.fw = 1; e.score = (int32_t)c.perfect; e.hasEdit = 0; e.pos = 0; e.chr = e.qchr = 0; e.pad[0] = e.pad[1] = 0; }
			if(tb[3] > tb[2]) { XEEHit &e = c.ee[c.nee++]; e.top = tb[2]; e.bot = tb[3]; e.fw = 0; e.score = (int32_t)c.perfect; e.hasEdit = 0; e.pos = 0; e.chr = e.qchr = 0; e.pad[0] = e.pad[1] = 0; }
		}
		if(u.nelt[0] > 0 && u.nelt[1] > 0 && u.nelt[0] > u.nelt[1]) { u.matemap[0] = 1; u.matemap[1] = 0; } else { u.matemap[0] = 0; u.matemap[1] = 1; }
		}
		for(u.mi = 0; u.mi < 2; u.mi++) {
			{
				const int mate = u.matemap[u.mi]; XMate &c = u.m[mate];
				if(u.nelt[mate] == 0) { c.nee = 0; continue; }
				if(x_ps_done_with_mate(u, mate == 0)) { c.nee = 0; u.done[mate] = 1; continue; }
				u.xAi = mate; u.xUseSh = 0; u.xUseEe = 1;
			}
			XE_CALL_EXT(1, stepExtPaired);
			{
				const int mate = u.matemap[u.mi]; XMate &c = u.m[mate];
				c.nee = 0;
				const int ret = u.xRet;
				if(ret == FULFILLED) { if(x_ps_done_with_mate(u, mate == 0)) u.done[mate] = 1; if(x_ps_done_with_mate(u, mate == 1)) u.done[mate ^ 1] = 1; }
				else if(ret == PERFECT || ret == HARD_LIMIT) u.done[mate] = 1;
				if(!u.done[mate] && c.minsc == c.perfect) u.done[mate] = 1;
			}
		}
		// ---- 1-mismatch end-to-end
		for(u.mi = 0; u.mi < 2; u.mi++) {
			{
				const int mate = u.matemap[u.mi]; XMate &c = u.m[mate];
				if(!c.filt || u.done[mate]) { c.nmm1 = 0; u.nelt[mate] = 0; continue; }
				u.nelt[mate] = 0;
				const bool yfw = u.mined[mate][0] <= 1 && !u.nofwM[mate], yrc = u.mined[mate][1] <= 1 && !u.norcM[mate];
				if(!(yfw || yrc)) continue;
				u.rqRead = c.idx; u.rqMinsc = (int32_t)c.minsc; u.rqNofw = !yfw; u.rqNorc = !yrc;
			}
			XE_WAIT(u.pc, 2, XR_ONE_MM);
			{
				const int mate = u.matemap[u.mi];
				loadMm1(u.m[mate], &u.nelt[mate]);
				if(u.fallback) return XR_FALLBACK;
			}
		}
		if(u.nelt[0] > 0 && u.nelt[1] > 0 && u.nelt[0] > u.nelt[1]) { u.matemap[0] = 1; u.matemap[1] = 0; } else { u.matemap[0] = 0; u.matemap[1] = 1; }
		for(u.mi = 0; u.mi < 2; u.mi++) {
			{
				const int mate = u.matemap[u.mi];
				if(u.nelt[mate] == 0) continue;
				if(x_ps_done_with_mate(u, mate == 0)) { u.done[mate] = 1; continue; }
				u.xAi = mate; u.xUseSh = 0; u.xUseEe = 0;
			}
			XE_CALL_EXT(3, stepExtPaired);
			{
				const int mate = u.matemap[u.mi]; XMate &c = u.m[mate];
				c.nmm1 = 0;
				const int ret = u.xRet;
				if(ret == FULFILLED) { if(x_ps_done_with_mate(u, mate == 0)) u.done[mate] = 1; if(x_ps_done_with_mate(u, mate == 1)) u.done[mate ^ 1] = 1; }
				else if(ret == PERFECT || ret == HARD_LIMIT) u.done[mate] = 1;
				if(!u.done[mate] && c.minsc == c.perfect) u.done[mate] = 1;
			}
		}
		// ---- seed rounds
		for(int k = 0; k < 2; k++) u.nrounds[k] = u.nroundsAll < u.interval[k] ? u.nroundsAll : u.interval[k];
		for(u.roundi = 0; u.roundi < P.seedRounds; u.roundi++) {
			u.m[0].hasSh = u.m[1].hasSh = 0;
			for(u.mi = 0; u.mi < 2; u.mi++) {
				{
					const int mate = u.matemap[u.mi]; XMate &c = u.m[mate];
					if(u.done[mate] || x_ps_done_with_mate(u, mate == 0)) { u.done[mate] = 1; continue; }
					if(u.roundi >= u.nrounds[mate] || u.interval[mate] <= u.roundi) continue;
					const int offset = (u.interval[mate] * u.roundi) / u.nrounds[mate];
					const int L = P.seedLen < c.rdlen ? P.seedLen : c.rdlen;
					if(offset > 0 && L + offset > c.rdlen) continue;
					u.rqRead = c.idx; u.rqL = L; u.rqInterval = u.interval[mate]; u.rqOffset = offset; u.rqNofw = u.nofwM[mate]; u.rqNorc = u.norcM[mate];
				}
				XE_WAIT(u.pc, 4, XR_SEED);
				{
					const int mate = u.matemap[u.mi]; XMate &c = u.m[mate];
					fillSeedHits(c, u.rqInterval, u.rqOffset, u.rqL);
					if(u.fallback) return XR_FALLBACK;
					if(c.shNonz == 0) { u.done[mate] = 1; break; }
					c.hasSh = 1;
				}
			}
			{
				double uniq[2] = {0.0, 0.0};
				for(int k = 0; k < 2; k++) if(u.m[k].hasSh) {
					for(int i = 0; i < u.m[k].shN; i++) { const int64_t x = shSize(u.m[k], true, i); if(x > 0) uniq[k] += 1.0 / (double)(x * x); }
					for(int i = 0; i < u.m[k].shN; i++) { const int64_t x = shSize(u.m[k], false, i); if(x > 0) uniq[k] += 1.0 / (double)(x * x); }
				}
				if(u.m[0].hasSh && u.m[1].hasSh && uniq[1] > uniq[0]) { u.matemap[0] = 1; u.matemap[1] = 0; } else { u.matemap[0] = 0; u.matemap[1] = 1; }
			}
			for(u.mi = 0; u.mi < 2; u.mi++) {
				{
					const int mate = u.matemap[u.mi]; XMate &c = u.m[mate];
					if(u.done[mate] || x_ps_done_with_mate(u, mate == 0)) { u.done[mate] = 1; continue; }
					if(!c.hasSh) continue;
					u.cur = mate;
					rankSeedHits(c);
					u.xAi = mate; u.xUseSh = 1; u.xUseEe = 0;
				}
				XE_CALL_EXT(5, stepExtPaired);
				{
					const int mate = u.matemap[u.mi];
					const int ret = u.xRet;
					if(ret == FULFILLED) { if(x_ps_done_with_mate(u, mate == 0)) u.done[mate] = 1; if(x_ps_done_with_mate(u, mate == 1)) u.done[mate ^ 1] = 1; }
					else if(ret == PERFECT || ret == HARD_LIMIT) u.done[mate] = 1;
				}
			}
			for(int k = 0; k < 2; k++) if(!u.done[k] && u.m[k].hasSh && u.m[k].shNelt / u.m[k].shNonz < 300) u.done[k] = 1;
		}
		finishPair();
		u.doneFlag = 1;
		return XR_DONE;
	}
	}
	XE_FB(u);
	return XR_FALLBACK;
}

// selectByScore over a list of (score, index): descending score, ties by descending index, then the reference's shuffle
// of equal-score streaks (aln_sink.cpp:1477-1628)
struct XSel { int64_t score; int32_t idx; };
XE_HD inline void x_select(XSel *buf, int n, XRng &rnd) {
	for(int i = 1; i < n; i++) {
		const XSel t = buf[i]; int j = i - 1;
		while(j >= 0 && (buf[j].score < t.score || (buf[j].score == t.score && buf[j].idx < t.idx))) { buf[j + 1] = buf[j]; j--; }
		buf[j + 1] = t;
	}
	int streak = 0;
	for(int i = 1; i < n; i++) {
		if(buf[i].score == buf[i - 1].score) { if(streak == 0) streak = 1; streak++; }
		else { if(streak > 1) x_shuffle_portion(buf, i - streak, streak, rnd); streak = 0; }
	}
	if(streak > 1) x_shuffle_portion(buf, n - streak, streak, rnd);
}
// -k / -a (Svc::kReport): the sink list(s) rearranged into the selected order (the report order of the secondaries), in place: buf[i].score is
// free once the caller has read the scores it needs; list b (a concordant pair's mate-2 list) is moved along with list a
XE_HD inline void x_permute_selected(XSel *buf, int n, uint16_t *a, uint16_t *b) {
	for(int i = 0; i < n; i++) buf[i].score = (int64_t)a[buf[i].idx] | (b ? (int64_t)b[buf[i].idx] << 16 : 0);
	for(int i = 0; i < n; i++) { a[i] = (uint16_t)buf[i].score; if(b) b[i] = (uint16_t)(buf[i].score >> 16); }
}

template <typename Svc>
XE_HD void XEngine<Svc>::finishPair() {
	u.pairType = 0; u.pairKind = 5; u.scoreSum = 0; u.fraglen = 0;
	for(int k = 0; k < 2; k++) { u.resAligned[k] = 0; u.resHasXs[k] = 0; u.resMapq[k] = 0; u.resXs[k] = 0; u.resAln[k] = 0xffff; }
	const int64_t mn[2] = {u.m[0].rdlen ? P.minScore(u.m[0].rdlen) : 0, u.m[1].rdlen ? P.minScore(u.m[1].rdlen) : 0};
	XSel buf[XE_LIST];
	if(u.nconcord > 0) {
		const int n = u.nrs12;
		for(int i = 0; i < n; i++) { buf[i].score = (int64_t)x_aln(u, u.rs1[i])->score + x_aln(u, u.rs2[i])->score; buf[i].idx = i; }
		x_select(buf, n, u.rnd);
		const uint16_t o1 = u.rs1[buf[0].idx], o2 = u.rs2[buf[0].idx];
		const XAln *a1 = x_aln(u, o1), *a2 = x_aln(u, o2);
		const bool hasC = n > 1;
		const int mq = (int)mapq((int64_t)a1->score + a2->score, hasC, hasC ? buf[1].score : 0, mn[0] + mn[1], u.m[0].perfect + u.m[1].perfect);
		for(int k = 0; k < 2; k++) {
			u.resAligned[k] = 1; u.resAln[k] = k == 0 ? o1 : o2; u.resMapq[k] = mq;
			const XAln *ch = k == 0 ? a1 : a2;
			const uint16_t *rsu = k == 0 ? u.rs1u : u.rs2u; const int nu = k == 0 ? u.nrs1u : u.nrs2u;
			bool has = false; int64_t best = 0;
			for(int i = 0; i < nu; i++) {
				const XAln *a = x_aln(u, rsu[i]);
				if(a->tidx == ch->tidx && a->refoff == ch->refoff && a->fw == ch->fw) continue;
				if(!has || a->score > best) { has = true; best = a->score; }
			}
			u.resHasXs[k] = has; u.resXs[k] = best;
		}
		u.pairType = 1;
		u.scoreSum = (int64_t)a1->score + a2->score;
		u.pairKind = pe_classify(P.pe, a1->refoff, (uint64_t)a1->refExtent(), a1->fw != 0, a2->refoff, (uint64_t)a2->refExtent(), a2->fw != 0);
		{   // fragment length (pe.cpp:89-92): the span of the two alignments, soft-trimmed ends included
			const int64_t s1 = a1->refoff - a1->trimLeft(), e1 = a1->refoff + a1->refExtent() + (a1->rdlen - a1->ext() - a1->trimLeft());
			const int64_t s2 = a2->refoff - a2->trimLeft(), e2 = a2->refoff + a2->refExtent() + (a2->rdlen - a2->ext() - a2->trimLeft());
			u.fraglen = (e1 > e2 ? e1 : e2) - (s1 < s2 ? s1 : s2);
		}
		if(Svc::kReport && !P.mmode) x_permute_selected(buf, n, u.rs1, u.rs2);
		return;
	}
	if(!u.doneDiscord && u.nunp[0] == 1 && u.nunp[1] == 1) {
		const XAln *a1 = x_aln(u, u.rs1u[0]), *a2 = x_aln(u, u.rs2u[0]);
		const int mq = (int)mapq((int64_t)a1->score + a2->score, false, 0, mn[0] + mn[1], u.m[0].perfect + u.m[1].perfect);
		for(int k = 0; k < 2; k++) { u.resAligned[k] = 1; u.resAln[k] = k == 0 ? u.rs1u[0] : u.rs2u[0]; u.resMapq[k] = mq; }
		u.pairType = 2;
		return;
	}
	int nal = 0;
	for(int k = 0; k < 2; k++) {
		const uint16_t *rsu = k == 0 ? u.rs1u : u.rs2u; const int nu = k == 0 ? u.nrs1u : u.nrs2u;
		if(nu == 0 || !P.mixed) continue;
		for(int i = 0; i < nu; i++) { buf[i].score = x_aln(u, rsu[i])->score; buf[i].idx = i; }
		x_select(buf, nu, u.rnd);
		u.resAligned[k] = 1; u.resAln[k] = rsu[buf[0].idx];
		u.resHasXs[k] = nu > 1; u.resXs[k] = nu > 1 ? x_aln(u, rsu[buf[1].idx])->score : 0;
		u.resMapq[k] = (int)mapq(x_aln(u, u.resAln[k])->score, u.resHasXs[k] != 0, u.resXs[k], mn[k], u.m[k].perfect);
		if(Svc::kReport && !P.mmode) x_permute_selected(buf, nu, k == 0 ? u.rs1u : u.rs2u, nullptr);
		nal++;
	}
	u.pairType = nal == 2 ? 2 : (nal == 1 ? 3 : 0);
}

// ---------------------------------------------------------------------------------------------- single reads
// multiseedSearchWorker for an unpaired read, as policy_engine.cpp: Engine::readSteps
template <typename Svc>
XE_HD int XEngine<Svc>::stepRead() {
	XMate &c = u.m[0];
	switch(u.pc) {
	case 0: {
		{
		const int idx = (int)u.id, len = svc.rdlen(idx);
		u.pairType = 0; u.pairKind = 5; u.scoreSum = 0; u.fraglen = 0;
		for(int k = 0; k < 2; k++) { u.resAligned[k] = 0; u.resHasXs[k] = 0; u.resMapq[k] = 0; u.resXs[k] = 0; u.resAln[k] = 0xffff; }
		if(len > P.maxLen) { XE_FB(u); return XR_FALLBACK; }
		c.idx = idx; c.rdlen = len;
		{
			const uint8_t *cd = svc.codes(idx);
			int ns = 0;
			for(int i = 0; i < len; i++) ns += cd[i] > 3;
			if(len < 2 || ns > P.nCeil(len) || P.perfect(len) < P.minScore(len)) { u.doneFlag = 1; return XR_DONE; }
		}
		c.minsc = P.minScore(len); c.perfect = P.perfect(len); c.nceil = P.nCeil(len); c.filt = 1;
		c.nee = c.nmm1 = c.hasSh = 0; c.nexr[0] = c.nexr[1] = 0; c.nseen = 0; c.nranks = 0; c.shN = 0; c.shNonz = c.shNelt = 0;
		u.rnd.init(svc.randSeed(idx));
		u.interval[0] = P.seedInterval(len, false);
		u.khits = P.khits; u.mhits = P.mhits;
		u.usDone = u.usExitM = u.usExitK = 0; u.usBest = u.usBest2 = XE_MIN_I64; u.nus = 0;
		u.nred[0] = u.nred[1] = u.nred[2] = 0;
		u.nIters = u.nDps = u.nUgs = u.nMateDps = 0;
		u.rdone = 0;
		{
			uint64_t tb[4]; int mined[2];
			svc.sweep(idx, mined, tb);
			if(P.nofw) { tb[0] = tb[1] = 0; mined[0] = 0; }
			if(P.norc) { tb[2] = tb[3] = 0; mined[1] = 0; }
			u.mined[0][0] = mined[0]; u.mined[0][1] = mined[1];
			u.nelt[0] = (int64_t)((tb[1] > tb[0] ? tb[1] - tb[0] : 0) + (tb[3] > tb[2] ? tb[3] - tb[2] : 0));
			if(tb[1] > tb[0]) { XEEHit &e = c.ee[c.nee++]; e.top = tb[0]; e.bot = tb[1]; e.fw = 1; e.score = (int32_t)c.perfect; e.hasEdit = 0; e.pos = 0; e.chr = e.qchr = 0; e.pad[0] = e.pad[1] = 0; }
			if(tb[3] > tb[2]) { XEEHit &e = c.ee[c.nee++]; e.top = tb[2]; e.bot = tb[3]; e.fw = 0; e.score = (int32_t)c.perfect; e.hasEdit = 0; e.pos = 0; e.chr = e.qchr = 0; e.pad[0] = e.pad[1] = 0; }
		}
		}
		if(u.nelt[0] > 0) {
			u.xUseSh = 0; u.xUseEe = 1;
			XE_CALL_EXT(1, stepExtUnpaired);
			c.nee = 0;
			if(u.xRet == FULFILLED) { if(u.usDone) u.rdone = 1; }
			else if(u.xRet == PERFECT || u.xRet == HARD_LIMIT) u.rdone = 1;
			if(!u.rdone && c.minsc == c.perfect) u.rdone = 1;
		}
		if(!u.rdone) {
			u.rqNofw = !(u.mined[0][0] <= 1 && !P.nofw); u.rqNorc = !(u.mined[0][1] <= 1 && !P.norc);
			if(!u.rqNofw || !u.rqNorc) {
				u.rqRead = c.idx; u.rqMinsc = (int32_t)c.minsc;
				XE_WAIT(u.pc, 2, XR_ONE_MM);
				loadMm1(c, nullptr);
				if(u.fallback) return XR_FALLBACK;
				if(c.nmm1 > 0 && !u.usDone) {
					u.xUseSh = 0; u.xUseEe = 0;
					XE_CALL_EXT(3, stepExtUnpaired);
					c.nmm1 = 0;
					if(u.xRet == FULFILLED) { if(u.usDone) u.rdone = 1; }
					else if(u.xRet == PERFECT || u.xRet == HARD_LIMIT) u.rdone = 1;
					if(!u.rdone && c.minsc == c.perfect) u.rdone = 1;
				} else if(c.nmm1 > 0) u.rdone = 1;
			}
		}
		u.nrounds[0] = P.seedRounds < u.interval[0] ? P.seedRounds : u.interval[0];
		for(u.roundi = 0; u.roundi < P.seedRounds; u.roundi++) {
			if(u.rdone || u.usDone) { u.rdone = 1; break; }
			if(u.roundi >= u.nrounds[0] || u.interval[0] <= u.roundi) continue;
			{
				const int offset = (u.interval[0] * u.roundi) / u.nrounds[0];
				const int L = P.seedLen < c.rdlen ? P.seedLen : c.rdlen;
				if(offset > 0 && L + offset > c.rdlen) continue;
				u.rqRead = c.idx; u.rqL = L; u.rqInterval = u.interval[0]; u.rqOffset = offset; u.rqNofw = P.nofw; u.rqNorc = P.norc;
			}
			XE_WAIT(u.pc, 4, XR_SEED);
			fillSeedHits(c, u.rqInterval, u.rqOffset, u.rqL);
			if(u.fallback) return XR_FALLBACK;
			if(c.shNonz == 0) { u.rdone = 1; break; }
			u.cur = 0;
			rankSeedHits(c);
			u.xUseSh = 1; u.xUseEe = 0;
			XE_CALL_EXT(5, stepExtUnpaired);
			if(u.xRet == FULFILLED) { if(u.usDone) u.rdone = 1; }
			else if(u.xRet == PERFECT || u.xRet == HARD_LIMIT) u.rdone = 1;
			if(!u.rdone && c.shNelt / c.shNonz < 300) u.rdone = 1;
		}
		finishRead();
		u.doneFlag = 1;
		return XR_DONE;
	}
	}
	XE_FB(u);
	return XR_FALLBACK;
}

template <typename Svc>
XE_HD void XEngine<Svc>::finishRead() {
	if(u.nus == 0) return;
	XSel buf[XE_LIST];
	for(int i = 0; i < u.nus; i++) { buf[i].score = x_aln(u, u.usAlns[i])->score; buf[i].idx = i; }
	x_select(buf, u.nus, u.rnd);
	u.resAligned[0] = 1; u.resAln[0] = u.usAlns[buf[0].idx];
	u.resHasXs[0] = u.nus > 1; u.resXs[0] = u.nus > 1 ? buf[1].score : 0;
	u.resMapq[0] = (int)mapq(x_aln(u, u.resAln[0])->score, u.resHasXs[0] != 0, u.resXs[0], P.minScore(u.m[0].rdlen), u.m[0].perfect);
	if(Svc::kReport && !P.mmode) x_permute_selected(buf, u.nus, u.usAlns, nullptr);
}

// one step of a unit: runs until the next batched request (returned) or the end (XR_DONE)
template <typename Svc>
XE_HD inline int x_step(const XParams &P, XUnit &u, Svc &svc) {
	XEngine<Svc> e(P, u, svc);
	const int r = u.paired ? e.stepPair() : e.stepRead();
	if(u.fallback) return XR_FALLBACK;
	return r;
}
XE_HD inline void x_unit_reset(XUnit &u, uint32_t id, bool paired) {
	u.pc = 0; u.pcExt = 0; u.fallback = 0; u.paired = paired; u.doneFlag = 0; u.id = id; u.arenaTop = 0; u.cur = 0;
	u.nents = 0; u.nsats = 0; u.nrands = 0; u.nseenPool = 0; u.nhitl = 0; u.natt = 0; u.attCursor = 0; u.dpSlot = -1;
	u.pairType = 0; u.pairKind = 5; u.scoreSum = 0; u.fraglen = 0;
	for(int k = 0; k < 2; k++) { u.resAligned[k] = 0; u.resHasXs[k] = 0; u.resMapq[k] = 0; u.resXs[k] = 0; u.resAln[k] = 0xffff; }
}

// one alignment (or none: an unaligned row) -> a row of the pipeline's result arrays (policy_engine.cpp: fillResult)
XE_HD inline void x_fill_row(const XAln *a, bool hasXs, int64_t xs, int mapq, const uint8_t *codes, bt2g_read_result &out, uint8_t *ops, uint32_t maxOps) {
	out.found = 0; out.score = 0; out.score2 = INT32_MIN; out.fw = 0; out.tidx = 0; out.refoff = 0; out.nops = 0; out.ndp = 0;
	out.trim_left = out.trim_right = 0; out.mapq = 0; out.pad = 0;
	if(!a) return;
	const int nops = x_aln_to_ops(a, codes, ops, maxOps);
	out.found = (a->nedits == 0 && a->ext() == a->rdlen) ? 2 : 1;
	out.score = a->score; if(hasXs) out.score2 = (int32_t)xs;
	out.fw = a->fw; out.tidx = (uint64_t)a->tidx; out.refoff = a->refoff; out.nops = nops;
	out.trim_left = a->trimLeft(); out.trim_right = a->rdlen - a->ext() - a->trimLeft();
	out.mapq = mapq; out.pad = a->refns;
}
// the primary of read k of a finished unit
XE_HD inline void x_fill_result(const XUnit &u, int k, const uint8_t *codes, bt2g_read_result &out, uint8_t *ops, uint32_t maxOps) {
	x_fill_row(u.resAligned[k] ? x_aln(u, u.resAln[k]) : nullptr, u.resHasXs[k] != 0, u.resXs[k], u.resMapq[k], codes, out, ops, maxOps);
}

// ---------------------------------------------------------------------------------------------- -k / -a report
// The entries of a finished unit in the layout of bt2g_policy_align_k / _pairs_k (policy_engine.cpp: the `finish` lambda of
// policyAlign).  With Svc::kReport, finishRead / finishPair leave the sink lists in report order outside -M mode, so secondary j of a list is its
// element j, and ReportingState::getReport (aln_sink.cpp:300-330) reports min(found, khits) of them, the primary included
// (after a -k short circuit found >= khits).  Under -M every unit reports its primaries only.
XE_HD inline int x_report_secondaries(const XUnit &u, const XParams &P, int n) {
	if(P.mmode || n < 1) return 0;
	return (int)((int64_t)n < P.khits ? (int64_t)n : P.khits) - 1;
}
// entries before any cap: unpaired, the primary and its secondaries (0 when unaligned: the unaligned row is written all the same);
// paired, see x_report_entry
XE_HD inline int x_report_count(const XUnit &u, const XParams &P) {
	if(!u.paired) return u.resAligned[0] ? 1 + x_report_secondaries(u, P, u.nus) : 0;
	if(u.pairType == 1) return 1 + x_report_secondaries(u, P, u.nrs12);
	const int s0 = u.resAligned[0] ? x_report_secondaries(u, P, u.nrs1u) : 0, s1 = u.resAligned[1] ? x_report_secondaries(u, P, u.nrs2u) : 0;
	if(s0 + s1 == 0) return 1;
	return (u.resAligned[0] ? 1 + s0 : 1) + (u.resAligned[1] ? 1 + s1 : 1);
}
// entry e of a finished unit: one row (unpaired) or two rows and a pair record (paired), ops rows of maxOps bytes.
// Paired entries: entry 0 = the primaries; after a concordant pair, the further concordant pairs (both rows secondary); else, when a
// mate has secondaries, every record of mate 1 and then of mate 2, each beside the opposite mate's primary, an unaligned mate's row
// last (AlnSinkWrap::finishRead, aln_sink.cpp:930-1010).  found bit 8: secondary (FLAG 256, MAPQ 255, the primary's XS:i);
// bit 9: the row is there only as its mate's mate.
XE_HD inline void x_report_entry(const XUnit &u, const XParams &P, int e, const uint8_t *codes0, const uint8_t *codes1, bt2g_read_result *res,
                                 uint8_t *ops, uint32_t maxOps, bt2g_pair_result *pr) {
	if(!u.paired) {
		if(e == 0) { x_fill_result(u, 0, codes0, res[0], ops, maxOps); return; }
		x_fill_row(x_aln(u, u.usAlns[e]), u.resHasXs[0] != 0, u.resXs[0], 255, codes0, res[0], ops, maxOps);
		res[0].found |= 0x100;
		return;
	}
	int which[2] = {0, 0}, mark[2] = {0, 0};              // which: 0 = the mate's primary, j > 0 = element j of its report list
	const uint16_t *list[2] = {u.rs1, u.rs2};
	if(u.pairType == 1) {
		if(e > 0) { which[0] = which[1] = e; mark[0] = mark[1] = 0x100; }
	} else {
		list[0] = u.rs1u; list[1] = u.rs2u;
		const int s0 = u.resAligned[0] ? x_report_secondaries(u, P, u.nrs1u) : 0, s1 = u.resAligned[1] ? x_report_secondaries(u, P, u.nrs2u) : 0;
		if(s0 + s1 > 0) {
			const int A = u.resAligned[0] ? 1 + s0 : 0, B = u.resAligned[1] ? 1 + s1 : 0;
			if(e < A) { mark[1] = 0x200; if(e > 0) { which[0] = e; mark[0] = 0x100; } }
			else if(e - A < B) { mark[0] = 0x200; if(e - A > 0) { which[1] = e - A; mark[1] = 0x100; } }
			else mark[u.resAligned[0] ? 0 : 1] = 0x200;      // the unaligned mate's own row, beside the aligned mate's primary
		}
	}
	const uint8_t *codes[2] = {codes0, codes1};
	for(int k = 0; k < 2; k++) {
		if(which[k]) x_fill_row(x_aln(u, list[k][which[k]]), u.resHasXs[k] != 0, u.resXs[k], 255, codes[k], res[k], ops + (size_t)k * maxOps, maxOps);
		else x_fill_result(u, k, codes[k], res[k], ops + (size_t)k * maxOps, maxOps);
		res[k].found |= mark[k];
	}
	pr->pair_type = u.pairType; pr->kind = u.pairKind; pr->source = 0; pr->score_sum = (int32_t)u.scoreSum; pr->fraglen = u.fraglen;
}

} // namespace xe
