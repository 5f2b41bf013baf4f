// dp_device.cuh -- launch descriptor shared by api.cu and dp_kernels.cu (DP types: include/bt2g.h)
#pragma once
#include "bt2g_internal.h"
#include <cstdlib>

// the s16x2 kernels need every reachable score within +-DPX_LIMIT (dp_kernels.cu): end-to-end mode,
// minimum score >= -8000 and perfect score <= 8000
static inline bool dp_packed_ok(const bt2g_scoring &sc, int64_t minMinsc, int maxLen) {
	return !sc.local && minMinsc >= -8000 && (int64_t)sc.match_bonus * maxLen <= 8000 && sc.match_bonus >= 0;
}

// DpLaunch.mode: 0 = k_dp_e2e (32-bit, move codes), 1 = k_dp_e2e_x2 (s16x2, move codes),
// 3 = k_dp_fill_h + k_dp_tail_h (s16x2, H bytes: needs perfect - (minsc - bonus - 1) <= 127 for every problem) over chunks of a
//     workspace of DpLaunch.chunk problems (chunk * codeStride bytes; chunks planned by dp_chunk_size).
// There is no mode 2 any more (a fused H-byte kernel, retired: DESIGN section 3).  `cap` (bt2g_ctx::dpModeCap, set by
// bt2g_set_dp_mode) caps the mode; a cap of 2 selects what a cap of 1 does.
static inline int dp_kernel_mode(const bt2g_scoring &sc, int64_t minMinsc, int maxLen, int cap = 3) {
	if(cap < 0 || cap > 3) cap = 3;
	if(cap == 0 || !dp_packed_ok(sc, minMinsc, maxLen)) return 0;
	const int64_t range = (int64_t)sc.match_bonus * maxLen - (minMinsc - sc.match_bonus - 1);
	return (cap == 3 && range <= 127) ? 3 : 1;
}

// rows per lane: the H-byte kernels (mode 3) take the smallest R of {4,5,6,8,10,12,16} with 32 R >= rdlen
// (a 150 bp read fills 30 lanes at R = 5 instead of 19 at R = 8); the move-code kernels use 4 / 8 / 16.
static inline int dp_rows_per_lane(int maxLen, int mode) {
	if(mode == 3) {
		const int rs[7] = {4, 5, 6, 8, 10, 12, 16};
		for(int i = 0; i < 7; i++) if(32 * rs[i] >= maxLen) return rs[i];
		return 0;
	}
	return maxLen <= 128 ? 4 : (maxLen <= 256 ? 8 : (maxLen <= 512 ? 16 : 0));
}
// Mode 3 fills row blocks of 32 lanes x DP_BLOCK_RPL rows (k_dp_fill_h); a block takes at most maxCol + 31 steps.
#define DP_BLOCK_RPL 2
// bytes of workspace per problem (per warp slot in modes 0, 1): (maxCol + 32) steps x 32 lanes x R rows; in mode 3 R rounds up
// to whole row blocks and a block has room for maxCol + 36 steps: the 5 steps per block the blocks leave free hold their range
// table and the up to 3 steps past the last block's end that the fill's last group of steps stores
static inline uint64_t dp_code_stride(int maxCol, int maxLen, int mode) {
	int R = dp_rows_per_lane(maxLen, mode);
	if(mode == 3) R = (R + DP_BLOCK_RPL - 1) / DP_BLOCK_RPL * DP_BLOCK_RPL;
	const uint64_t steps = (uint64_t)maxCol + (mode == 3 ? 36 : 32);
	return ((steps * 32 * (uint64_t)R) + 255) & ~(uint64_t)255;   // 256 B aligned
}

// mode 3 workspace: as many problems as fit a byte budget (BT2G_DP_CHUNK_MB overrides it), at least 1024
static inline uint64_t dp_chunk_problems(uint64_t codeStride, uint64_t nMax, uint64_t budget) {
	if(const char *e = getenv("BT2G_DP_CHUNK_MB")) { uint64_t v = strtoull(e, nullptr, 10); if(v) budget = v << 20; }
	uint64_t c = budget / (codeStride ? codeStride : 1);
	if(c < 1024) c = 1024;
	if(c > nMax) c = nMax;
	return c ? c : 1;
}

// mode 3 chunk planning: a queue of n problems through a workspace (or half of one) of cap problems runs as k = ceil(n / cap)
// chunks of equal size rather than full chunks and a small remainder, each rounded up to whole rounds of the fill (`round`:
// the problems its resident warps hold at once) where cap allows: a chunk of 2.2 rounds takes as long as one of 3
static inline uint64_t dp_chunk_size(uint64_t n, uint64_t cap, uint64_t round) {
	if(cap < 1) cap = 1;
	const uint64_t k = (n + cap - 1) / cap;
	uint64_t c = k ? (n + k - 1) / k : cap;
	if(round) { const uint64_t r = (c + round - 1) / round * round; if(r <= cap) c = r; }
	return c ? c : 1;
}

struct DpLaunch {
	const uint8_t  *seq, *qual;
	const uint64_t *roff;
	const bt2g_dp_problem *probs;
	uint64_t        n;
	const uint32_t *nDev;         // optional: problem count produced on the device
	uint64_t        numSlots;     // persistent warp slots (multiple of 4)
	uint8_t        *codes;        // workspace (DpPlan::codeBytes): codeStride bytes per warp slot (mode 0), per problem of a slot's
	                              // pair (mode 1) or per problem of a chunk (mode 3)
	uint64_t       *rawKeys = nullptr;  // local mode: per-slot candidate keys (score<<32 | row<<16 | col)
	int             maxRaw = 0;   // local mode: keys per slot in rawKeys
	uint64_t        codeStride;
	int             maxCol;
	int             maxCands, maxAlns, maxOps;
	uint64_t        chunk = 0;    // mode 3: problems the workspace holds (dp_chunk_problems); chunks are planned by dp_chunk_size
	int             mode = 0;     // e2e: the kernel generation (dp_kernel_mode)
	uint32_t       *taskCtr = nullptr;  // mode 3 (required): 4 device words, the fill's and the tail's task counters of either half
	cudaStream_t    st2 = nullptr;      // mode 3, optional: consecutive chunks alternate between the launch's stream and st2, each in
	cudaEvent_t     evFork = nullptr, evJoin = nullptr;   // its own half of the workspace (st2 first waits for, then joins, the stream)
	uint64_t       *nChunks = nullptr;  // mode 3, optional: chunks launched (a fill and a tail each)
	cudaEvent_t    *tev = nullptr;  // optional timing marks (mode 3): before the fill, between fill and tail, after the tail of every chunk
	int             tevCap = 0;
	int            *tevN = nullptr;
	uint32_t        zeroP = 0;    // always 0: a zero the compiler cannot see through, so that it stays in ONE register (a literal 0 as
	                              // the third operand of VIADDMNMX is re-materialised with a PRMT before every use: 13 per step)
	bt2g_dp_summary *summ;
	bt2g_dp_cand    *cands;
	bt2g_dp_aln     *alns;
	uint8_t         *ops;
};

// The plan of one DP queue: the kernel generation and the workspace it needs.  numSlots: persistent warp slots; nMax: the most
// problems one launch takes; maxRaw: candidate keys per slot under local scoring; cap: the mode cap (bt2g_set_dp_mode);
// budget: the bytes a mode-3 workspace may take.
struct DpPlan {
	int      mode = 0;          // dp_kernel_mode; 0 under local scoring (k_dp_local)
	uint64_t codeStride = 0;    // dp_code_stride
	uint64_t chunk = 0;         // mode 3: problems the workspace holds (dp_chunk_problems)
	uint64_t codeBytes = 0;     // the move-code / H-byte workspace (DpLaunch::codes)
	bool     taskCtr = false;   // mode 3: 4 task-counter words (DpLaunch::taskCtr)
	int      maxRaw = 0;        // local: candidate keys per slot (DpLaunch::maxRaw)
	uint64_t rawKeys = 0;       // local: keys of all slots (DpLaunch::rawKeys)
};
static inline DpPlan dp_plan(const bt2g_scoring &sc, int64_t minMinsc, int maxLen, int maxCol, uint64_t nMax, uint64_t numSlots,
                             int maxRaw, int cap, uint64_t budget) {
	DpPlan P;
	P.mode = sc.local ? 0 : dp_kernel_mode(sc, minMinsc, maxLen, cap);
	P.codeStride = dp_code_stride(maxCol, maxLen, P.mode);
	if(P.mode == 3) {
		P.chunk = dp_chunk_problems(P.codeStride, nMax, budget);
		P.codeBytes = P.chunk * P.codeStride;
		P.taskCtr = true;
	} else {
		P.codeBytes = numSlots * P.codeStride * (P.mode ? 2 : 1);
	}
	if(sc.local) { P.maxRaw = maxRaw; P.rawKeys = numSlots * (uint64_t)maxRaw; }
	return P;
}
