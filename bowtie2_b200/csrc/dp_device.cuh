// dp_device.cuh -- launch descriptor shared by api.cu and dp_kernels.cu (DP types: include/bt2g.h)
#pragma once
#include "bt2g_internal.h"
#include <cstdlib>

// the s16x2 kernel needs every reachable score within +-DPX_LIMIT (dp_kernels.cu): end-to-end mode,
// minimum score >= -8000 and perfect score <= 8000; BT2G_DP_PACKED=0 in the environment disables it
static inline bool dp_packed_ok(const bt2g_scoring &sc, int64_t minMinsc, int maxLen) {
	return !sc.local && minMinsc >= -8000 && (int64_t)sc.match_bonus * maxLen <= 8000 && sc.match_bonus >= 0;
}

// DpLaunch.packed: 0 = k_dp_e2e (32-bit, move codes), 1 = k_dp_e2e_x2 (s16x2, move codes),
// 2 = k_dp_e2e_h (s16x2, H bytes: needs perfect - (minsc - bonus - 1) <= 127 for every problem),
// 3 = the same split into k_dp_fill_h + k_dp_tail_h over chunks of a workspace of DpLaunch.chunk problems
//     (chunk * codeStride bytes; chunks planned by dp_chunk_size).
// `cap` (bt2g_ctx::dpModeCap, set by bt2g_set_dp_mode; initialised once from BT2G_DP_PACKED at bt2g_create) caps the mode.
static inline int dp_kernel_mode(const bt2g_scoring &sc, int64_t minMinsc, int maxLen, int cap = 3) {
	if(cap < 0 || cap > 3) cap = 3;
	if(cap == 0 || !dp_packed_ok(sc, minMinsc, maxLen)) return 0;
	const int64_t range = (int64_t)sc.match_bonus * maxLen - (minMinsc - sc.match_bonus - 1);
	return (cap >= 2 && range <= 127) ? (cap >= 3 ? 3 : 2) : 1;
}

// rows per lane: the H-byte kernels (modes 2, 3) take the smallest R of {4,5,6,8,10,12,16} with 32 R >= rdlen
// (a 150 bp read fills 30 lanes at R = 5 instead of 19 at R = 8); the move-code kernels use 4 / 8 / 16.
static inline int dp_rows_per_lane(int maxLen, int mode) {
	if(mode >= 2) {
		const int rs[7] = {4, 5, 6, 8, 10, 12, 16};
		for(int i = 0; i < 7; i++) if(32 * rs[i] >= maxLen) return rs[i];
		return 0;
	}
	return maxLen <= 128 ? 4 : (maxLen <= 256 ? 8 : (maxLen <= 512 ? 16 : 0));
}
// Mode 3 fills row blocks of 32 lanes x DP_BLOCK_RPL rows (k_dp_fill_h); a block takes at most maxCol + 31 steps.
#define DP_BLOCK_RPL 2
// bytes of workspace per problem (per warp slot in modes 0-2): (maxCol + 32) steps x 32 lanes x R rows; in mode 3 R rounds up
// to whole row blocks and a block has room for maxCol + 36 steps: the 5 steps per block the blocks leave free hold their range
// table and the up to 3 steps past the last block's end that the fill's last group of steps stores
static inline uint64_t dp_code_stride(int maxCol, int maxLen, int mode) {
	int R = dp_rows_per_lane(maxLen, mode);
	if(mode == 3) R = (R + DP_BLOCK_RPL - 1) / DP_BLOCK_RPL * DP_BLOCK_RPL;
	const uint64_t steps = (uint64_t)maxCol + (mode == 3 ? 36 : 32);
	return ((steps * 32 * (uint64_t)R) + 255) & ~(uint64_t)255;   // planes of hb_index, 256 B aligned
}

// mode 3 workspace: as many problems as fit a byte budget (default 6 GiB; BT2G_DP_CHUNK_MB overrides), at least 1024
static inline uint64_t dp_chunk_problems(uint64_t codeStride, uint64_t nMax, uint64_t budget = 6ull << 30) {
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
	uint8_t        *codes;        // workspace: n * codeStride bytes
	int32_t        *lastH;
	uint64_t       *rawKeys;      // local mode: per-slot candidate keys (score<<32 | row<<16 | col)
	int             maxRaw;        // workspace: n * maxCol ints (e2e last-row scores)
	uint64_t        codeStride;
	int             maxCol;
	int             maxCands, maxAlns, maxOps;
	uint64_t        chunk = 0;    // mode 3: problems the workspace holds (dp_chunk_problems); chunks are planned by dp_chunk_size
	int             packed = 0;   // e2e: two problems per warp as s16x2 pairs (codes workspace: 2 * codeStride per slot)
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
