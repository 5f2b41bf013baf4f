// xengine_host.cpp -- the state machine of xengine.cuh driven on the HOST over a bt2g_policy_backend table: every request of a
// unit is answered at once with a batch-of-one call of the table's entry point.  This is not a product path (the product runs
// the same state machine as a kernel, csrc/xengine.cu); it exists so that the CPU test-suite can pin xengine.cuh against the
// reference program's SAM with the oracle answering behind the table, exactly as it pins csrc/policy_engine.cpp, and it
// supplies the pieces both drivers share: parameter tables, read seeds, result conversion.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/bt2g.h"
#define __host__
#define __device__
#define __forceinline__ inline
#include "xengine.cuh"
#include "xengine_shared.h"

namespace xe {

// ---- parameter resolution (policy_engine.cpp: policyAlign) with the SimpleFunc values tabulated per read length
static double funcF(int type, double C, double L, double x) {
	const double g = type == 1 ? 0.0 : type == 2 ? x : type == 3 ? std::sqrt(x) : std::log(x);
	return C + L * g;
}

void buildParams(const bt2g_policy_params *pp, int offSize, int maxLen, XParams &P, XTables &T) {
	memset(&P, 0, sizeof(P));
	P.local = pp->local; P.paired = pp->paired; P.all = pp->all_hits; P.mmode = pp->mmode; P.nofw = pp->nofw; P.norc = pp->norc;
	P.discord = pp->discord; P.mixed = pp->mixed;
	P.seedLen = pp->seed_len; P.seedRounds = pp->seed_rounds; P.streak = pp->dp_fail_streak;
	P.maxIters = 400; P.maxUg = 300; P.maxDp = 300; P.maxMateStreak = 10;
	P.khits = P.all ? XE_BIG : (pp->khits > 0 ? pp->khits : 1);
	P.mhits = P.mmode ? (pp->mhits > 0 ? pp->mhits : 50) : XE_BIG;
	if(P.all) { P.maxIters = P.maxUg = P.maxDp = P.streak = P.maxMateStreak = (int)(XE_BIG >> 33); }
	else if(P.khits > 1) { const int k1 = (int)(P.khits - 1); P.streak += k1 * 10; P.maxMateStreak += k1 * 10; P.maxIters += k1 * 20; P.maxUg += k1 * 20; P.maxDp += k1 * 20; }
	P.seed = pp->seed; P.offSize = offSize;
	P.matchBonus = pp->match_bonus; P.mmpMax = pp->mmp_max; P.mmpMin = pp->mmp_min; P.nPen = pp->n_pen;
	P.rdgConst = pp->rdgap_const; P.rdgLin = pp->rdgap_linear; P.rfgConst = pp->rfgap_const; P.rfgLin = pp->rfgap_linear;
	P.pe = pp->pe;
	if(maxLen > XE_MAX_LEN) maxLen = XE_MAX_LEN;
	P.maxLen = maxLen;
	T.minsc.assign(maxLen + 1, 0); T.nceilRaw.assign(maxLen + 1, 0); T.ivalOne.assign(maxLen + 1, 1); T.ivalBoth.assign(maxLen + 1, 1);
	for(int len = 1; len <= maxLen; len++) {
		const long long m = (long long)funcF(pp->smin_type, pp->smin_const, pp->smin_coeff, (double)len);
		T.minsc[len] = (int32_t)(P.local ? (m > 0 ? m : 0) : (m < 0 ? m : 0));
		T.nceilRaw[len] = (int32_t)(long long)funcF(2, pp->nceil_const, pp->nceil_coeff, (double)len);
		long long v = (long long)funcF(pp->ival_type, pp->ival_const, pp->ival_coeff, (double)len);
		T.ivalOne[len] = (int32_t)(v > 1 ? v : 1);
		long long vb = (long long)((double)v * 1.2 + 0.5);
		T.ivalBoth[len] = (int32_t)(vb > 1 ? vb : 1);
	}
	P.minscTab = T.minsc.data(); P.nceilRawTab = T.nceilRaw.data(); P.ivalOneTab = T.ivalOne.data(); P.ivalBothTab = T.ivalBoth.data();
}

// the device scoring scheme that corresponds to the policy's parameters (Scoring::initPens, scoring.h:103-132)
void scoringFromParams(const bt2g_policy_params *pp, bt2g_scoring *sc) {
	memset(sc, 0, sizeof(*sc));
	sc->match_bonus = pp->match_bonus;
	sc->rdgap_const = pp->rdgap_const; sc->rdgap_linear = pp->rdgap_linear; sc->rfgap_const = pp->rfgap_const; sc->rfgap_linear = pp->rfgap_linear;
	sc->gapbar = 4; sc->local = pp->local ? 1 : 0;
	for(int q = 0; q < 64; q++) {
		const int ii = q < 40 ? q : 40;
		const float frac = (float)ii / 40.0f;
		sc->mmpen[q] = (uint8_t)(pp->mmp_min + (int)(frac * (float)(pp->mmp_max - pp->mmp_min)));
		sc->npen[q] = (uint8_t)pp->n_pen;
	}
	sc->nceil_const = pp->nceil_const; sc->nceil_linear = pp->nceil_coeff;
}

uint32_t genRandSeed(const uint8_t *codes, const uint8_t *quals, int len, const char *name, uint32_t seed) {   // pat.cpp:45-82
	uint32_t rseed = (seed + 101u) * 59u * 61u * 67u * 71u * 73u * 79u * 83u;
	for(int i = 0; i < len; i++) rseed ^= (uint32_t)codes[i] << ((i & 15) << 1);
	for(int i = 0; i < len; i++) rseed ^= (uint32_t)quals[i] << ((i & 3) << 3);
	for(size_t i = 0; name && name[i]; i++) { if(name[i] == '/') break; rseed ^= (uint32_t)(unsigned char)name[i] << ((i & 3) << 3); }
	return rseed;
}

// ---- the services of xengine.cuh answered through the entry-point table, one item per call
struct HostSvc {
	static constexpr bool kReport = true;             // (the -M results do not depend on the order of the sink lists)
	const bt2g_policy_backend &be; const XParams &P; const bt2g_reads *reads; const char *const *names;
	int rc = 0; uint64_t nCalls = 0;
	// answers of the batched requests of the unit in flight
	std::vector<bt2g_mm_hit> mmHitsBuf; int32_t mmCounts[4] = {0, 0, 0, 0}; static constexpr int MH = 64;
	std::vector<uint64_t> seedOut[2]; int seedN[2] = {0, 0}, seedStride[2] = {1, 1};
	struct Dp { bt2g_dp_summary summ; std::vector<bt2g_dp_cand> cands; std::vector<bt2g_dp_aln> alns; std::vector<uint8_t> ops; int maxOps = 0; } dp[2];
	int maxCands = 1024, maxAlns = 16;
	std::vector<uint8_t> stretch; int64_t stTidx = -1, stOff = 0;
	HostSvc(const bt2g_policy_backend &b, const XParams &p, const bt2g_reads *r, const char *const *n) : be(b), P(p), reads(r), names(n) {}

	const uint8_t *codes(int read) const { return reads->seq + reads->off[read]; }
	const uint8_t *quals(int read) const { return reads->qual + reads->off[read]; }
	int rdlen(int read) const { return (int)(reads->off[read + 1] - reads->off[read]); }
	uint32_t randSeed(int read) const { return genRandSeed(codes(read), quals(read), rdlen(read), names ? names[read] : nullptr, P.seed); }
	bt2g_reads one(int read, uint64_t off2[2]) const {
		bt2g_reads b; b.n_reads = 1; b.seq = codes(read); b.qual = quals(read); off2[0] = 0; off2[1] = (uint64_t)rdlen(read); b.off = off2;
		return b;
	}
	void sweep(int read, int mined[2], uint64_t tb[4]) {
		uint64_t o2[2]; bt2g_reads b = one(read, o2);
		uint8_t mine[2] = {0, 0};
		rc |= be.exact_sweep(be.ctx, &b, 0, 0, mine, tb); nCalls++;
		mined[0] = mine[0]; mined[1] = mine[1];
	}
	void answerOneMm(const XUnit &u) {
		uint64_t o2[2]; bt2g_reads b = one(u.rqRead, o2);
		mmHitsBuf.assign((size_t)4 * MH, bt2g_mm_hit{});
		const int32_t minsc = u.rqMinsc; const uint8_t mask = (uint8_t)((u.rqNofw ? 0 : 1) | (u.rqNorc ? 0 : 2));
		rc |= be.one_mm(be.ctx, &b, &minsc, &mask, MH, mmHitsBuf.data(), mmCounts); nCalls++;
	}
	int mmMax() const { return MH; }
	int mmCount(int, int task) const { return mmCounts[task]; }
	const bt2g_mm_hit *mmHits(int, int task) const { return mmHitsBuf.data() + (size_t)task * MH; }
	void answerSeed(const XUnit &u) {
		const int read = u.rqRead, k = read & 1;
		uint64_t o2[2]; bt2g_reads b = one(read, o2);
		const int len = rdlen(read);
		int n = 1; if(len - u.rqOffset > u.rqL) n += (len - u.rqOffset - u.rqL) / u.rqInterval;
		const int nsMax = n + 2;
		const int32_t iv = u.rqInterval, of = u.rqOffset;
		bt2g_seed_plan plan{u.rqL, nsMax, u.rqNofw, u.rqNorc, &iv, &of};
		seedOut[k].assign((size_t)2 * nsMax * 4, 0);
		int32_t ns = 0;
		rc |= be.seed_search(be.ctx, &b, &plan, seedOut[k].data(), &ns); nCalls++;
		seedN[k] = ns; seedStride[k] = nsMax;
	}
	int nSeeds(int read) const { return seedN[read & 1]; }
	const uint64_t *seedRange(int read, int strand, int i) const { const int k = read & 1; return seedOut[k].data() + ((size_t)strand * seedStride[k] + i) * 4; }
	void answerDp(const XUnit &u, bool mate) {
		Dp &d = dp[mate ? 1 : 0];
		const int read = (int)u.rqProb.read_idx;
		uint64_t o2[2]; bt2g_reads b = one(read, o2);
		bt2g_dp_problem p = u.rqProb; p.read_idx = 0;
		int mc = P.local ? 16384 : maxCands, ma = maxAlns;
		for(int attempt = 0; attempt < 2; attempt++) {
			d.maxOps = rdlen(read) + 80;
			d.cands.assign((size_t)mc, bt2g_dp_cand{}); d.alns.assign((size_t)ma, bt2g_dp_aln{}); d.ops.assign((size_t)ma * d.maxOps, 0);
			rc |= be.dp_extend(be.ctx, &b, &p, 1, mc, ma, d.maxOps, &d.summ, d.cands.data(), d.alns.data(), d.ops.data()); nCalls++;
			if(!d.summ.flags) break;
			mc = 65536; ma = 128;                       // rare: more candidates / alignments than the first buffers hold
		}
		curMaxAlns = ma;
	}
	int curMaxAlns = 16;
	const bt2g_dp_summary *dpSumm(int, bool mate) const { return &dp[mate ? 1 : 0].summ; }
	const bt2g_dp_cand *dpCands(int, bool mate) const { return dp[mate ? 1 : 0].cands.data(); }
	const bt2g_dp_aln *dpAlns(int, bool mate) const { return dp[mate ? 1 : 0].alns.data(); }
	const uint8_t *dpOps(int, bool mate, int k) const { const Dp &d = dp[mate ? 1 : 0]; return d.ops.data() + (size_t)k * d.maxOps; }
	int dpMaxAlns() const { return curMaxAlns; }
	bool resolve(uint64_t row, int qlen, bool reject, int64_t &tidx, int64_t &toff, int64_t &tlen) {
		uint64_t joined = 0, ti = 0, to = 0, tl = 0; uint8_t fl = 0; const uint32_t hl = (uint32_t)qlen;
		rc |= be.resolve(be.ctx, &row, &hl, 1, reject ? 1 : 0, &joined, &ti, &to, &tl, &fl); nCalls++;
		tidx = (int64_t)ti; toff = (int64_t)to; tlen = (int64_t)tl;
		return !((fl >> 1) & 1);
	}
	void extend(int read, bool fw, int rdoff, int seedlen, const uint64_t rng[4], int &nlex, int &nrex) {
		uint64_t o2[2]; bt2g_reads b = one(read, o2);
		const int32_t iv = rdlen(read) > 1 ? rdlen(read) : 1, of = rdoff;
		bt2g_seed_plan plan{seedlen, 1, 0, 0, &iv, &of};
		uint64_t ranges[8] = {0, 0, 0, 0, 0, 0, 0, 0};
		for(int j = 0; j < 4; j++) ranges[(fw ? 0 : 1) * 4 + j] = rng[j];
		uint8_t out[4] = {0, 0, 0, 0};
		rc |= be.extend_exact(be.ctx, &b, &plan, ranges, out); nCalls++;
		nlex = out[(fw ? 0 : 1) * 2]; nrex = out[(fw ? 0 : 1) * 2 + 1];
	}
	int ungapped(int read, bool fw, int64_t tidx, int64_t refoff, int64_t tlen, int64_t minsc, bt2g_ungapped_result &r) {
		uint64_t o2[2]; bt2g_reads b = one(read, o2);
		bt2g_ungapped_problem p{}; p.read_idx = 0; p.fw = fw; p.tidx = (uint64_t)tidx; p.refoff = refoff; p.reflen = (uint64_t)tlen; p.minsc = (int32_t)minsc; p.ohang = 0;
		rc |= be.ungapped(be.ctx, &b, &p, 1, &r, nullptr, 0); nCalls++;
		if(r.status == 1) {
			const int32_t cnt = rdlen(read);
			stretch.assign((size_t)cnt, 4);
			const uint64_t ti = (uint64_t)tidx;
			rc |= be.get_stretch(be.ctx, &ti, &refoff, &cnt, 1, cnt, stretch.data()); nCalls++;
			stTidx = tidx; stOff = refoff;
		}
		return r.status;
	}
	int refChar(int64_t tidx, int64_t off) const {
		const int64_t k = off - stOff;
		if(tidx != stTidx || k < 0 || k >= (int64_t)stretch.size()) return 4;
		return stretch[(size_t)k];
	}
};

} // namespace xe

// internal entry of policy_engine.cpp: the coroutine engine on a sub-batch (fallback for units that outgrow the fixed state)
extern "C" int bt2g_policy_align(const bt2g_policy_backend *, const bt2g_policy_params *, const bt2g_reads *, const char *const *,
                                 bt2g_read_result *, uint8_t *, uint32_t, bt2g_pair_result *, uint64_t *);

// maxPer = 0: one row per read (bt2g_xengine_align_host); maxPer >= 1: the entry layout of bt2g_policy_align_k / _pairs_k with
// nEntries[unit] (bt2g_xengine_align_host_k).  Returns 1 when a unit had more entries than maxPer > 1.
static int alignHost(const bt2g_policy_backend *be, const bt2g_policy_params *pp, const bt2g_reads *reads, const char *const *names, uint32_t maxPer,
                     bt2g_read_result *res, uint8_t *ops, uint32_t maxOps, bt2g_pair_result *pairs, uint32_t *nEntries, uint64_t *stats) {
	using namespace xe;
	if(!be || !pp || !reads || !res || !ops || (pp->paired && (!pairs || (reads->n_reads & 1))) || (maxPer && !nEntries)) return -1;
	bool truncated = false;
	int maxLen = 1;
	for(uint64_t i = 0; i < reads->n_reads; i++) { const int l = (int)(reads->off[i + 1] - reads->off[i]); if(l > maxLen) maxLen = l; }
	XParams P; XTables T;
	buildParams(pp, be->off_size, maxLen, P, T);
	HostSvc svc(*be, P, reads, names);
	const size_t units = P.paired ? reads->n_reads / 2 : reads->n_reads;
	std::vector<XUnit> ubuf(1);
	XUnit &u = ubuf[0];
	uint64_t nReq = 0, nFallback = 0;
	for(size_t id = 0; id < units; id++) {
		x_unit_reset(u, (uint32_t)id, P.paired != 0);
		int r;
		for(;;) {
			r = x_step(P, u, svc);
			if(r == XR_DONE || r == XR_FALLBACK) break;
			nReq++;
			if(r == XR_ONE_MM) svc.answerOneMm(u);
			else if(r == XR_SEED) svc.answerSeed(u);
			else if(r == XR_DP) svc.answerDp(u, false);
			else if(r == XR_DP_MATE) svc.answerDp(u, true);
			u.dpSlot = 0;
			if(svc.rc) return -2;
		}
		if(svc.rc) return -2;
		const size_t r0 = P.paired ? 2 * id : id, nr = P.paired ? 2 : 1;
		if(r == XR_FALLBACK) {
			nFallback++;
			bt2g_reads sub; sub.n_reads = nr; sub.seq = reads->seq + reads->off[r0]; sub.qual = reads->qual + reads->off[r0];
			uint64_t off3[3] = {0, reads->off[r0 + 1] - reads->off[r0], nr == 2 ? reads->off[r0 + 2] - reads->off[r0] : 0};
			sub.off = off3;
			const char *nm[2] = {names ? names[r0] : nullptr, (names && nr == 2) ? names[r0 + 1] : nullptr};
			if(maxPer) {
				const size_t e0 = id * (size_t)maxPer;
				const int rc2 = P.paired ? bt2g_policy_align_pairs_k(be, pp, &sub, names ? nm : nullptr, maxPer, res + 2 * e0, ops + 2 * e0 * (size_t)maxOps, maxOps, pairs + e0, nEntries + id, nullptr)
				                         : bt2g_policy_align_k(be, pp, &sub, names ? nm : nullptr, maxPer, res + e0, ops + e0 * (size_t)maxOps, maxOps, nEntries + id, nullptr);
				if(rc2 < 0) return rc2;
				truncated = truncated || rc2 == 1;
				continue;
			}
			bt2g_pair_result pr{};
			const int rc2 = bt2g_policy_align(be, pp, &sub, names ? nm : nullptr, res + r0, ops + r0 * (size_t)maxOps, maxOps, P.paired ? &pr : nullptr, nullptr);
			if(rc2 < 0) return rc2;
			if(P.paired) pairs[id] = pr;
			continue;
		}
		if(maxPer) {
			// the same report function as the device engine's k_xe_report, one entry at a time
			const int n = x_report_count(u, P), nw = n < (int)maxPer ? n : (int)maxPer;
			truncated = truncated || (n > (int)maxPer && maxPer > 1);
			const size_t e0 = id * (size_t)maxPer;
			const uint8_t *c0 = svc.codes((int)r0), *c1 = P.paired ? svc.codes((int)r0 + 1) : nullptr;
			for(int e = 0; e < (nw > 1 ? nw : 1); e++)
				x_report_entry(u, P, e, c0, c1, res + (e0 + e) * nr, ops + (e0 + e) * nr * (size_t)maxOps, maxOps, P.paired ? pairs + e0 + e : nullptr);
			nEntries[id] = (uint32_t)nw;
			continue;
		}
		for(size_t k = 0; k < nr; k++) x_fill_result(u, (int)k, svc.codes((int)(r0 + k)), res[r0 + k], ops + (r0 + k) * (size_t)maxOps, maxOps);
		if(P.paired) {
			pairs[id] = bt2g_pair_result{}; pairs[id].pair_type = u.pairType; pairs[id].kind = u.pairKind;
			pairs[id].score_sum = (int32_t)u.scoreSum; pairs[id].fraglen = u.fraglen;
		}
	}
	if(stats) { stats[0] = units; stats[1] = nFallback; stats[2] = nReq; }
	return truncated ? 1 : 0;
}

extern "C" int bt2g_xengine_align_host(const bt2g_policy_backend *be, const bt2g_policy_params *pp, const bt2g_reads *reads, const char *const *names,
                                       bt2g_read_result *res, uint8_t *ops, uint32_t maxOps, bt2g_pair_result *pairs, uint64_t *stats) {
	return alignHost(be, pp, reads, names, 0, res, ops, maxOps, pairs, nullptr, stats);
}

extern "C" int bt2g_xengine_align_host_k(const bt2g_policy_backend *be, const bt2g_policy_params *pp, const bt2g_reads *reads, const char *const *names,
                                         uint32_t maxPerUnit, bt2g_read_result *res, uint8_t *ops, uint32_t maxOps, bt2g_pair_result *pairs,
                                         uint32_t *nEntries, uint64_t *stats) {
	if(maxPerUnit == 0 || !nEntries) return -1;
	return alignHost(be, pp, reads, names, maxPerUnit, res, ops, maxOps, pairs, nEntries, stats);
}
