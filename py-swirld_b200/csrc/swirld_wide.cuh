// swirld_wide.cuh -- the consensus kernels for ANY member count (member sets as NJ = ceil(M/32)
// 32-bit words): configs 4 and 5 of BASELINE.json (256 and 1024 members), and -- with SW_FORCE_WIDE=1 -- an
// independent second implementation of the M <= 64 path for A/B parity on the reference fixtures.
//
// Same math as swirld_kernels.cuh / swirld_rounds.cuh (DESIGN.md section 3), different machinery:
//
//   * "how many members c have a mask with bit c_" (the strongly-sees count of swirld.py:207-214 and
//     245-252) is a VERTICAL population count over up to M masks of M bits.  A lane owns one 32-bit word
//     (32 columns) of every mask and adds the masks into a bit-sliced counter with a Harley-Seal
//     carry-save tree: 16 masks cost 15 CSAs + one ripple into the upper planes, ~6 integer ops per mask
//     word; the threshold test `hits > 2T/3` is a bit-sliced compare, the promotion count a popcount.
//     For M < 1024 the 32 lanes are split into 32/NJ groups that take different members and the groups'
//     counters are added at the end.
//   * rounds: the monotone predicate P_r of swirld_rounds.cuh, one cooperative kernel, per step
//     (a) masks S_r(k) of the events the tests can meet (per-event cache with an exact (launch, round) tag),
//     grid barrier, (b) one warp per (chain, pending position) tests P_r, grid barrier, (c) identical
//     bookkeeping in every CTA.  With several GPUs (sw_peer_connect) the tests of a step are sharded by
//     chain and every rank writes its chains' first hits straight into every peer's buffer over NVLink
//     (P2P stores + a system-scope flag per source rank): compute and exchange in ONE kernel, no NCCL call
//     on the data path.
//   * decide_fame: a thread per undecided witness keeps its vote mask (NJ words) in registers; the voters'
//     strongly-seen sets are staged 32 at a time.
//   * find_order: per-chain received-threshold by bisection over the event index, consensus time by a
//     radix select over the seers' timestamps.
#pragma once
#include "swirld_kernels.cuh"

#define RW_THREADS 512
#define RW_RING 256          // == RB_RING: per-member ring of the events that precede the chunk
#define RW_LMAX 32
#define VC_PLANES 12         // bit-sliced counters hold up to 4095

// ------------------------------------------------------------------ bit-sliced vertical counter
#define VC_CSA(h, l, a, b, c) { const unsigned _u = (a) ^ (b); h = ((a) & (b)) | (_u & (c)); l = _u ^ (c); }

struct VCounter {
    unsigned ones, twos, fours, eights;
    unsigned up[VC_PLANES - 4];          // weights 16, 32, ...
    __device__ __forceinline__ void clear() {
        ones = twos = fours = eights = 0;
#pragma unroll
        for (int i = 0; i < VC_PLANES - 4; i++) up[i] = 0;
    }
    __device__ __forceinline__ void add16(const unsigned (&x)[16]) {
        unsigned tA, tB, fA, fB, eA, eB, sx;
        VC_CSA(tA, ones, ones, x[0], x[1]); VC_CSA(tB, ones, ones, x[2], x[3]); VC_CSA(fA, twos, twos, tA, tB);
        VC_CSA(tA, ones, ones, x[4], x[5]); VC_CSA(tB, ones, ones, x[6], x[7]); VC_CSA(fB, twos, twos, tA, tB);
        VC_CSA(eA, fours, fours, fA, fB);
        VC_CSA(tA, ones, ones, x[8], x[9]); VC_CSA(tB, ones, ones, x[10], x[11]); VC_CSA(fA, twos, twos, tA, tB);
        VC_CSA(tA, ones, ones, x[12], x[13]); VC_CSA(tB, ones, ones, x[14], x[15]); VC_CSA(fB, twos, twos, tA, tB);
        VC_CSA(eB, fours, fours, fA, fB);
        VC_CSA(sx, eights, eights, eA, eB);
#pragma unroll
        for (int i = 0; i < VC_PLANES - 4; i++) { const unsigned t = up[i] & sx; up[i] ^= sx; sx = t; }
    }
    __device__ __forceinline__ unsigned plane(int p) const {
        return p == 0 ? ones : p == 1 ? twos : p == 2 ? fours : p == 3 ? eights : up[p - 4];
    }
    __device__ __forceinline__ void set_plane(int p, unsigned v) {
        if (p == 0) ones = v; else if (p == 1) twos = v; else if (p == 2) fours = v; else if (p == 3) eights = v; else up[p - 4] = v;
    }
    // this += the counter held by lane ^ d
    __device__ __forceinline__ void add_lane_xor(int d) {
        unsigned carry = 0;
#pragma unroll
        for (int p = 0; p < VC_PLANES; p++) {
            const unsigned a = plane(p), b = __shfl_xor_sync(0xffffffffu, a, d);
            const unsigned u = a ^ b;
            set_plane(p, u ^ carry);
            carry = (a & b) | (u & carry);
        }
    }
    // columns whose count is > thr (thr < 2^VC_PLANES)
    __device__ __forceinline__ unsigned greater_than(unsigned thr) const {
        unsigned gt = 0, eq = 0xffffffffu;
#pragma unroll
        for (int p = VC_PLANES - 1; p >= 0; p--) {
            const unsigned v = plane(p);
            if ((thr >> p) & 1) eq &= v;
            else { gt |= eq & v; eq &= ~v; }
        }
        return gt;
    }
};

// The columns c_ with  sum over members m with ev[m] >= 0 of stake[m] * [bit c_ of mask(ev[m])]  >  thr.
// ev: M ints in shared memory (-1 = the member contributes nothing); masks: [event][NJ] words in global memory.
// Returns, in lane w < NJ, word w of the result (32 columns).  UNIT: stake 1 per member (bit-sliced path).
template <int NJ>
__device__ __forceinline__ unsigned vcount_gt(const int *ev, int M, const unsigned *__restrict__ masks, i64 thr,
                                              bool unit, const i64 *stake, int lane) {
    constexpr int G = 32 / NJ;                    // lane groups working on different members
    const int g = lane / NJ, w = lane % NJ;
    if (unit) {
        VCounter vc;
        vc.clear();
        const int iters = (M + G - 1) / G;
        auto fetch = [&](int it0, unsigned (&x)[16]) {
#pragma unroll
            for (int u = 0; u < 16; u++) {
                const int m = (it0 + u) * G + g;
                const int k = (it0 + u < iters && m < M) ? ev[m] : -1;
                x[u] = k >= 0 ? __ldcg(masks + (size_t)k * NJ + w) : 0u;
            }
        };
        // two batches of 16 mask words in flight: the next one is fetched before the current one is added
        unsigned xa[16], xb[16];
        fetch(0, xa);
        for (int it0 = 0; it0 < iters; it0 += 32) {
            if (it0 + 16 < iters) fetch(it0 + 16, xb);
            vc.add16(xa);
            if (it0 + 16 < iters) {
                if (it0 + 32 < iters) fetch(it0 + 32, xa);
                vc.add16(xb);
            }
        }
#pragma unroll
        for (int d = NJ; d < 32; d <<= 1) vc.add_lane_xor(d);
        if (thr >= (1 << VC_PLANES) - 1) return 0u;
        return vc.greater_than((unsigned)thr);
    }
    // integer stakes: every lane group walks all members for its own 32/G... simple and exact, rarely used
    unsigned out = 0;
    for (int b = g; b < 32; b += G) {            // column 32*w + b
        i64 acc = 0;
        for (int m = 0; m < M; m++) {
            const int k = ev[m];
            if (k >= 0 && ((__ldcg(masks + (size_t)k * NJ + w) >> b) & 1)) acc += stake[m];
        }
        if (acc > thr) out |= 1u << b;
    }
#pragma unroll
    for (int d = NJ; d < 32; d <<= 1) out |= __shfl_xor_sync(0xffffffffu, out, d);
    return out;
}

// masks: {c_ : W[c_] >= 0 and row(k)[c_] >= W[c_]} as NJ words; lane w < NJ returns word w.  Wc in shared memory.
template <int NJ>
__device__ __forceinline__ unsigned seen_words(const int32_t *__restrict__ rowk, const int *Wc, int M, int lane) {
    unsigned mine = 0;
    int v[NJ];
#pragma unroll
    for (int j = 0; j < NJ; j++) v[j] = lane + 32 * j < M ? __ldcg(rowk + lane + 32 * j) : -1;      // the whole row in flight at once
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        const int c = lane + 32 * j;
        const int wv = c < M ? Wc[c] : -1;
        const unsigned b = __ballot_sync(0xffffffffu, wv >= 0 && v[j] >= wv);
        if (lane == j) mine = b;
    }
    return mine;
}

// ------------------------------------------------------------------ rounds (divide_rounds, swirld.py:187-222)
struct RwParams {
    int M, first, n, Rcap, L;
    unsigned epoch;
    const int32_t *row, *p0, *creator, *seq;
    int32_t *round;
    int32_t *Wf;                // [Rcap][M]
    unsigned *scw;              // [cap][NJ] mask cache
    u64 *sctag;                 // [cap] (epoch << 32 | round + 1) of the cached mask
    int32_t *cev;               // chunk events grouped by creator at [first, first+n) (k_rb_prep, like cmin, coff, ctot, bar)
    int32_t *cmin, *coff, *ctot, *gchain;
    unsigned *bar;
    u64 *hitmin;                // [3][M]
    unsigned *ticket;           // [3] work counter of a step's tests (cleared like hitmin)
    const i64 *stake;
    i64 tot2;
    int unit;
    int32_t *scal;
    // several GPUs: tests sharded by chain (chain % nranks == rank), first hits written to every peer
    int rank, nranks;
    u64 *xhit[8];               // peer p's exchange buffer: [nranks (source)][3][M]
    unsigned *xflag[8];         // peer p's flags: [nranks (source)] = steps published by that source
    unsigned *xstep;            // steps this rank has published so far (flags count steps for ever; device-resident
                                // because the step count of a launch is data dependent)
    long long *dbg;
};

__device__ __forceinline__ void rw_grid_barrier(unsigned *ctr, unsigned &target) {
    __syncthreads();
    target += gridDim.x;
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0) { __threadfence(); atomicAdd(ctr, 1u); }
        __syncwarp();
        unsigned v;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while ((int)(v - target) < 0);
        __syncwarp();
    }
    __syncthreads();
}

__device__ __forceinline__ u64 rw_tag(int r, unsigned epoch) { return ((u64)epoch << 32) | (unsigned)(r + 1); }

// publish S_r(k) (lane w < NJ holds word w) with its tag; readers: tag first (acquire), then the words
template <int NJ>
__device__ __forceinline__ void rw_publish(const RwParams &P, int k, unsigned word, u64 tag, int lane, bool fence = true) {
    if (lane < NJ) P.scw[(size_t)k * NJ + lane] = word;
    if (fence) __threadfence();          // (not needed when a grid barrier separates the producers from the readers)
    __syncwarp();
    if (lane == 0) {
        if (fence) asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(P.sctag + k), "l"(tag) : "memory");
        else asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(P.sctag + k), "l"(tag) : "memory");
    }
}
__device__ __forceinline__ u64 rw_ld_tag(const u64 *p) {
    u64 v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ u64 rw_ld_tag_relaxed(const u64 *p) {      // (the producer is a grid barrier away)
    u64 v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

template <int NJ>
__global__ void __launch_bounds__(RW_THREADS, 1) k_rounds_wide(RwParams P) {
    extern __shared__ int rw_smem[];
    const int M = P.M;
    // chain state, identical in every CTA (and on every rank)
    i64 *stake_s = reinterpret_cast<i64 *>(rw_smem);    // [M]
    int *cur = rw_smem + 2 * M, *pos = cur + M, *len = pos + M, *off = len + M, *cmin_s = off + M, *ctot_s = cmin_s + M;
    int *Wc = ctot_s + M, *Wn = Wc + M;                 // Wf of the current round and of the next one
    int *lo_ev = Wn + M, *hi_ev = lo_ev + M;            // first / last event of a member whose S_r mask is prepared
    int *rlo = hi_ev + M, *rbase = rlo + M;             // masks to prepare this step: start seq, exclusive prefix of the counts (rbase[M] = total)
    int *s_nfin = rbase + M + 1, *s_base = s_nfin + M;
    int *pdone = s_base + M;                            // seq up to which a member's masks of round rprev are prepared (this launch)
    int *ntest = pdone + M;                             // pending positions of the member tested this step
    int *red = ntest + M;                               // [32] reduction scratch
    int *spre_all = red + 32;                           // [warps][M] per-warp staging of a test's pre[] row
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gw = blockIdx.x * (RW_THREADS / 32) + warp, nw = gridDim.x * (RW_THREADS / 32);
    const bool lead = blockIdx.x == 0;
    const i64 thr = P.tot2 / 3;
    const bool unit = P.unit != 0;
    int *spre = spre_all + (size_t)warp * M;
    u64 *xmine = P.nranks > 1 ? P.xhit[P.rank] : nullptr;   // my own exchange buffer (what the peers wrote for me)

    auto block_min = [&](int v) -> int {                // min over the CTA (all threads call it)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
        __syncthreads();
        if (lane == 0) red[warp] = v;
        __syncthreads();
        v = red[0];
        for (int w2 = 1; w2 < RW_THREADS / 32; w2++) v = min(v, red[w2]);
        return v;
    };

    int rtop = max(P.scal[SC_MAX_ROUND], 0);
    const unsigned xbase = (P.nranks > 1 && lead) ? *P.xstep : 0u;      // (written back by CTA 0 after the last barrier)
    for (int c = tid; c < M; c += RW_THREADS) {
        stake_s[c] = P.stake[c];
        const int o = P.first + P.coff[c], l = P.coff[c + 1] - P.coff[c];
        int cu = 0x7fffffff;
        if (l > 0) { const int h0 = P.cev[o], pa = P.p0[h0]; cu = pa < 0 ? 0 : P.round[pa]; }
        off[c] = o; len[c] = l; pos[c] = 0; cur[c] = cu;
        cmin_s[c] = P.cmin[c]; ctot_s[c] = P.ctot[c];
        if (l > 0 && cu == 0) {                         // a member's root opens round 0 for it
            const int h0 = P.cev[o];
            if (P.p0[h0] < 0 && lead) P.Wf[c] = h0;
        }
    }
    if (lead) for (int i = tid; i < 3 * M; i += RW_THREADS) P.hitmin[i] = ~0ull;
    if (lead && tid < 3) P.ticket[tid] = 0;
    long long cyc[6] = {0, 0, 0, 0, 0, 0}, c_tests = 0, c_full = 0, c_tmax = 0;
    unsigned bar_target = 0;
    rw_grid_barrier(P.bar, bar_target);                 // roots are in the global table, hitmin is clear

    int rprev = -2;                                     // round whose Wf rows sit in Wc / Wn
    bool abort_all = false;
    unsigned step = 0;
    for (;; ++step) {
        const long long t0 = clock64();
        // ---- lowest open round
        int rmin = 0x7fffffff;
        for (int c = tid; c < M; c += RW_THREADS) if (pos[c] < len[c]) rmin = min(rmin, cur[c]);
        rmin = block_min(rmin);
        if (rmin == 0x7fffffff) break;
        if (rmin >= P.Rcap - 1) { if (lead && tid == 0) atomicMin(&P.scal[SC_ERR], -5); break; }
        // ---- Wf rows of rmin and rmin+1.  Only row rmin+1 is written during this launch (by the bookkeeping below,
        //      mirrored in Wn by every CTA), so any other row can be read from the global table without a race.
        if (rmin != rprev) {
            for (int c = tid; c < M; c += RW_THREADS) {
                const int keep = Wn[c];
                Wc[c] = (rmin == rprev + 1) ? keep : __ldcg(P.Wf + (size_t)rmin * M + c);
                Wn[c] = __ldcg(P.Wf + (size_t)(rmin + 1) * M + c);
                pdone[c] = 0;
            }
            rprev = rmin;
        }
        // ---- the step's frontier: the pending events of the chains at rmin with an index below X are tested, and the
        //      masks S_rmin of EVERY event below X are prepared first -- a tested event sees nothing at or above itself,
        //      so every mask a test needs is there (nothing is left to chance or deferred)
        int xmin = 0x7fffffff;
        for (int c = tid; c < M; c += RW_THREADS)
            if (pos[c] < len[c] && cur[c] == rmin) xmin = min(xmin, P.cev[off[c] + pos[c]]);
        xmin = block_min(xmin);
        const int X = xmin + P.L * M;
        const int buf = step % 3;
        const u64 tag = rw_tag(rmin, P.epoch);
        for (int c = tid; c < M; c += RW_THREADS) {
            // tested positions of this chain: its pending events below X (at most RW_LMAX)
            int nt = 0, nbelow;
            const bool active = pos[c] < len[c] && cur[c] == rmin;
            const int32_t *ce = P.cev + off[c];
            if (active) {
                int a = 0, b = min(RW_LMAX, len[c] - pos[c]);
                while (a < b) { const int mid = (a + b) >> 1; if (ce[pos[c] + mid] < X) a = mid + 1; else b = mid; }
                nt = a;
            }
            ntest[c] = nt;
            {   // the member's events of this chunk below X
                int a = active ? pos[c] + nt : 0, b = len[c];
                if (active && nt < min(RW_LMAX, len[c] - pos[c])) b = a;
                while (a < b) { const int mid = (a + b) >> 1; if (ce[mid] < X) a = mid + 1; else b = mid; }
                nbelow = a;
            }
            int lo = 0, cnt = 0, le = 0x7fffffff, he = -1;
            const int w = Wc[c];
            if (w >= 0) {
                lo = __ldcg(P.seq + w);
                const int before = len[c] > 0 ? cmin_s[c] : ctot_s[c];      // seq of the member's first event of this chunk
                if (lo < before) lo = max(lo, before - RW_RING);            // older events are not in the ring any more
                const int hi = len[c] > 0 ? cmin_s[c] + nbelow : ctot_s[c];
                const int start = max(lo, pdone[c]);                        // [lo, start) was prepared by earlier steps of this round
                cnt = max(0, min(hi - start, RW_RING));
                pdone[c] = start + cnt;
                if (start + cnt > lo) {
                    auto ev_at = [&](int sq) -> int {
                        if (len[c] > 0 && sq >= cmin_s[c]) return ce[sq - cmin_s[c]];
                        return __ldcg(P.gchain + (size_t)c * RW_RING + (sq & (RW_RING - 1)));
                    };
                    le = ev_at(lo); he = ev_at(start + cnt - 1);
                }
                lo = start;
            }
            rlo[c] = lo; rbase[c] = cnt; lo_ev[c] = le; hi_ev[c] = he;
        }
        __syncthreads();
        if (warp == 0) {                                // exclusive scan of the counts
            const int per = (M + 31) / 32;
            const int b0 = lane * per, b1 = min(M, b0 + per);
            int sacc = 0;
            for (int c = b0; c < b1; c++) sacc += rbase[c];
            int inc = sacc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
            int run = inc - sacc;
            for (int c = b0; c < b1; c++) { const int v = rbase[c]; rbase[c] = run; run += v; }
            if (lane == 31) rbase[M] = inc;
        }
        __syncthreads();
        const long long t1 = clock64();
        {   // ---- (a) masks of the new events below the frontier
            const int total = rbase[M];
            for (int i = gw; i < total; i += nw) {
                int a = 0, b = M;                       // member whose range holds candidate i: last c with rbase[c] <= i
                while (b - a > 1) { const int mid = (a + b) >> 1; if (rbase[mid] <= i) a = mid; else b = mid; }
                const int c = a, sq = rlo[c] + (i - rbase[c]);
                int k;
                if (len[c] > 0 && sq >= cmin_s[c]) k = P.cev[off[c] + sq - cmin_s[c]];
                else k = __ldcg(P.gchain + (size_t)c * RW_RING + (sq & (RW_RING - 1)));
                if (k < 0) continue;
                if (rw_ld_tag_relaxed(P.sctag + k) == tag) continue;  // prepared by an earlier step of this round
                const unsigned word = seen_words<NJ>(P.row + (size_t)k * M, Wc, M, lane);
                rw_publish<NJ>(P, k, word, tag, lane, false);
            }
        }
        const long long t2 = clock64();
        rw_grid_barrier(P.bar, bar_target);
        const long long t3 = clock64();
        // ---- (b) tests: one warp per (chain, tested position); with several ranks, my share of the chains
        {
            // work items: (my chain, tested position) pairs, handed out by a ticket counter (a test that ends at the
            // cheap live-stake check frees its warp for the next one)
            const int nown = (M - P.rank + P.nranks - 1) / P.nranks;
            for (;;) {
                unsigned tk = 0;
                if (lane == 0) tk = atomicAdd(P.ticket + buf, 1u);
                const int i = (int)__shfl_sync(0xffffffffu, tk, 0);
                if (i >= nown * RW_LMAX) break;
                const int tc = (i / RW_LMAX) * P.nranks + P.rank, tj = i % RW_LMAX;
                if (tj >= ntest[tc]) continue;
                const long long tt0 = clock64();
                const int th = P.cev[off[tc] + pos[tc] + tj];
                const int tpa = P.p0[th];
                if (tpa < 0) continue;                                  // a root is never promoted
                i64 lv = 0;
                __syncwarp();
                int rv[NJ];
#pragma unroll
                for (int j = 0; j < NJ; j++) rv[j] = lane + 32 * j < M ? __ldcg(P.row + (size_t)th * M + lane + 32 * j) : -1;   // the row in flight at once
#pragma unroll
                for (int j = 0; j < NJ; j++) {
                    const int c = lane + 32 * j;
                    if (32 * j >= M) break;
                    int v = -1;
                    bool live = false;
                    if (c < M) {
                        v = c == tc ? tpa : rv[j];
                        const int wv = Wc[c];
                        live = wv >= 0 && v >= wv;
                        spre[c] = live ? v : -1;
                    }
                    if (unit) lv += __popc(__ballot_sync(0xffffffffu, live));
                    else {
                        i64 sacc = live ? stake_s[c] : 0;
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
                        lv += sacc;
                    }
                }
                __syncwarp();
                c_tests++;
                if (lv <= thr) continue;                                // hits[c_] <= stake of the live members
                // a mask outside the prepared ranges (an event older than the ring): checked by tag, computed here
                for (int c0 = 0; c0 < M; c0 += 32) {
                    const int c = c0 + lane;
                    const int k = c < M ? spre[c] : -1;
                    bool miss = false;
                    if (k >= 0 && (k < lo_ev[c] || k > hi_ev[c])) miss = rw_ld_tag(P.sctag + k) != tag;
                    unsigned mm = __ballot_sync(0xffffffffu, miss);
                    while (mm) {
                        const int l = __ffs(mm) - 1;
                        mm &= mm - 1;
                        const int kk = __shfl_sync(0xffffffffu, k, l);
                        const unsigned word = seen_words<NJ>(P.row + (size_t)kk * M, Wc, M, lane);
                        rw_publish<NJ>(P, kk, word, tag, lane);
                    }
                }
                __syncwarp();
                const unsigned gt = vcount_gt<NJ>(spre, M, P.scw, thr, unit, stake_s, lane);
                int cnt = lane < NJ ? __popc(gt) : 0;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
                if ((i64)cnt > thr && lane == 0) atomicMin(P.hitmin + (size_t)buf * M + tc, ((u64)tj << 32) | (unsigned)th);
                const long long dt = clock64() - tt0;
                c_full++; c_tmax = dt > c_tmax ? dt : c_tmax;
            }
        }
        const long long t4 = clock64();
        rw_grid_barrier(P.bar, bar_target);
        const long long t5 = clock64();
        // ---- several GPUs: my chains' first hits go to every rank (P2P stores over NVLink), then one flag per peer
        const u64 *hsrc = P.hitmin + (size_t)buf * M;
        if (P.nranks > 1) {
            if (lead) {
                for (int c = P.rank + P.nranks * tid; c < M; c += P.nranks * RW_THREADS) {
                    const u64 v = __ldcg(hsrc + c);
                    for (int p = 0; p < P.nranks; p++) P.xhit[p][((size_t)P.rank * 3 + buf) * M + c] = v;
                }
                __threadfence_system();
                __syncthreads();
                const unsigned want = xbase + step + 1;
                if (tid < P.nranks)
                    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(P.xflag[tid] + P.rank), "r"(want) : "memory");
                if (tid < P.nranks) {
                    const long long t0 = clock64();
                    unsigned v;
                    for (;;) {
                        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(P.xflag[P.rank] + tid) : "memory");
                        if ((int)(v - want) >= 0) break;
                        if (clock64() - t0 > 8000000000ll) { atomicMin(&P.scal[SC_ERR], -4); break; }   // ~4 s: a peer is gone
                    }
                }
                __syncthreads();
            }
            rw_grid_barrier(P.bar, bar_target);
            if (__ldcg(P.scal + SC_ERR) == -4) abort_all = true;
        }
        if (abort_all) break;
        // ---- (c) identical bookkeeping in every CTA (only CTA 0 writes the global tables)
        bool opened = false;
        for (int c = tid; c < M; c += RW_THREADS) {
            int nfinal = 0, o = 0;
            if (ntest[c] > 0) {
                const u64 hm = P.nranks > 1 ? __ldcg(xmine + ((size_t)(c % P.nranks) * 3 + buf) * M + c) : __ldcg(hsrc + c);
                o = off[c] + pos[c];
                if (hm != ~0ull) {
                    const int ft = (int)(hm >> 32), hnew = (int)(unsigned)hm;
                    nfinal = ft;                        // the events before the first hit are final at rmin
                    cur[c] = rmin + 1;
                    Wn[c] = hnew;
                    if (lead) P.Wf[(size_t)(rmin + 1) * M + c] = hnew;
                    opened = true;
                } else nfinal = ntest[c];
                pos[c] += nfinal;
            }
            s_nfin[c] = nfinal; s_base[c] = o;
        }
        if (__syncthreads_or(opened)) rtop = max(rtop, rmin + 1);
        if (lead) {                                     // clear the buffer the step after next will use
            const int nb2 = (buf + 2) % 3;
            for (int c = tid; c < M; c += RW_THREADS) P.hitmin[(size_t)nb2 * M + c] = ~0ull;
            if (tid == 0) P.ticket[nb2] = 0;
        }
        for (int i = blockIdx.x + gridDim.x * tid; i < M * RW_LMAX; i += gridDim.x * RW_THREADS) {
            const int c = i / RW_LMAX, j = i % RW_LMAX;
            if (j < s_nfin[c]) P.round[P.cev[s_base[c] + j]] = rmin;
        }
        __syncthreads();
        const long long t6 = clock64();
        cyc[0] += t1 - t0; cyc[1] += t2 - t1; cyc[2] += t3 - t2; cyc[3] += t4 - t3; cyc[4] += t5 - t4; cyc[5] += t6 - t5;
    }
    if (P.dbg && lane == 0) {            // profiling counters (tools/rounds_cycles.py): [0..5] setup, masks, barrier, tests, barrier(+exchange), bookkeeping
        unsigned long long *o = (unsigned long long *)P.dbg;
        if (lead && warp == 0) { for (int i = 0; i < 6; i++) atomicAdd(&o[i], (unsigned long long)cyc[i]); atomicAdd(&o[6], (unsigned long long)step); }
        atomicAdd(&o[9], (unsigned long long)c_tests); atomicAdd(&o[10], (unsigned long long)c_full);
        atomicMax(&o[8], (unsigned long long)c_tmax);
    }
    if (lead && tid == 0 && P.n > 0) P.scal[SC_MAX_ROUND] = rtop;
    if (lead && tid == 0 && P.nranks > 1) *P.xstep = xbase + step;
}

// ---- SM(h) = {c_ : W[round h][c_] >= 0 and row(h)[c_] >= W[round h][c_]} as NJ words, one warp per event
template <int NJ>
__global__ void __launch_bounds__(256) k_w_seenmask(int M, int first, int n, int Rcap, const int32_t *row, const int32_t *round,
                                                    const int32_t *W, unsigned *SMw) {
    const int lane = threadIdx.x & 31;
    const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = gridDim.x * (blockDim.x >> 5);
    for (int j0 = gw; j0 < n; j0 += nw) {
        const int h = first + j0, r = round[h];
        unsigned mine = 0;
        if (r >= 0 && r < Rcap) {
            const int32_t *Wr = W + (size_t)r * M;
            int v[NJ], w[NJ];
#pragma unroll
            for (int j = 0; j < NJ; j++) {
                const int c = lane + 32 * j;
                v[j] = c < M ? row[(size_t)h * M + c] : -1;
                w[j] = c < M ? Wr[c] : -1;
            }
#pragma unroll
            for (int j = 0; j < NJ; j++) {
                const unsigned b = __ballot_sync(0xffffffffu, w[j] >= 0 && v[j] >= w[j]);
                if (lane == j) mine = b;
            }
        }
        if (lane < NJ) SMw[(size_t)h * NJ + lane] = mine;
    }
}

// ---- decide_fame's strongly-seen set s(y) of every new witness (swirld.py:245-254, quirk Q15)
template <int NJ>
__global__ void __launch_bounds__(256) k_w_strong(StrongParams P) {
    extern __shared__ int sw_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, M = P.M;
    i64 *stake_s = reinterpret_cast<i64 *>(sw_smem);                 // [M]
    int *ev = sw_smem + 2 * M + (size_t)warp * M;
    for (int c = threadIdx.x; c < M; c += blockDim.x) stake_s[c] = P.stake[c];
    __syncthreads();
    const int gw = blockIdx.x * (blockDim.x >> 5) + warp, nw = gridDim.x * (blockDim.x >> 5);
    const int cnt = *P.list_n;
    for (int i = gw; i < cnt; i += nw) {
        const int h = P.list[i];
        if (!P.wit[h]) continue;
        const int rh = P.round[h];
        if (rh < 0 || rh >= P.Rcap) continue;
        const int ch = P.creator[h];
        if (lane == 0) P.coin[(size_t)rh * M + ch] = P.sig[(size_t)h * 64] >> 7;
        if (rh < 1) continue;
        const int r = rh - 1;
        __syncwarp();
        {
            int k[NJ], rk[NJ];
#pragma unroll
            for (int j = 0; j < NJ; j++) k[j] = lane + 32 * j < M ? P.row[(size_t)h * M + lane + 32 * j] : -1;
#pragma unroll
            for (int j = 0; j < NJ; j++) rk[j] = k[j] >= 0 ? P.round[k[j]] : -1;
#pragma unroll
            for (int j = 0; j < NJ; j++) if (lane + 32 * j < M) ev[lane + 32 * j] = (k[j] >= 0 && rk[j] == r) ? k[j] : -1;
        }
        __syncwarp();
        const unsigned gt = vcount_gt<NJ>(ev, M, P.SMw, P.tot2 / 3, P.unit != 0, stake_s, lane);
        if (lane < NJ) P.Sw[((size_t)rh * M + ch) * NJ + lane] = gt;
    }
}

// ------------------------------------------------------------------ decide_fame (swirld.py:224-277)
template <int NJ>
__device__ __forceinline__ i64 w_wsum(const unsigned (&m)[NJ], bool unit, const i64 *stake_s) {
    i64 s = 0;
#pragma unroll
    for (int w = 0; w < NJ; w++) {
        unsigned x = m[w];
        if (unit) s += __popc(x);
        else while (x) { const int b = __ffs(x) - 1; s += stake_s[32 * w + b]; x &= x - 1; }
    }
    return s;
}

// One THREAD per witness x = (r, mx): its vote mask over the voters of the previous voter round (NJ words) stays in
// registers; the voters' sets S[r_][m] are staged 32 voters at a time.  A candidate round r is spread over
// ceil(M / FW_THREADS) CTAs (the witnesses are independent recurrences); they add up rem[r] / done[r], which
// k_fame_begin cleared.
#define FW_THREADS 256
template <int NJ>
__device__ __forceinline__ void w_fame_rounds_body(const FameParams &P) {
    extern __shared__ int fw_smem[];
    unsigned *sS = reinterpret_cast<unsigned *>(fw_smem);            // [32][NJ] staged voter sets
    int *vw = fw_smem + 32 * NJ;                                     // [32] voter present
    int *vcoin = vw + 32;                                            // [32]
    i64 *vsum = reinterpret_cast<i64 *>(vcoin + 32);                 // [32] stake of the voter's set
    i64 *stake_s = vsum + 32;                                        // [M]
    const int tid = threadIdx.x, M = P.M;
    const int parts = (M + FW_THREADS - 1) / FW_THREADS, mx = (blockIdx.x % parts) * FW_THREADS + tid;
    const bool unit = P.unit != 0;
    const int max_r = P.scal[SC_MAX_ROUND], max_c = P.scal[SC_MAXC];
    for (int c = tid; c < M; c += blockDim.x) stake_s[c] = P.stake[c];
    for (int r = max_c + blockIdx.x / parts; r <= max_r; r += gridDim.x / parts) {
        __syncthreads();
        const size_t slot = (size_t)r * M + mx;
        int x = -1;
        bool live = false;
        if (!P.consensus[r] && mx < M) { x = P.W[slot]; live = x >= 0 && P.famous[slot] < 0; }
        bool any_decided = false;
        unsigned pv[NJ];
#pragma unroll
        for (int w = 0; w < NJ; w++) pv[w] = 0;
        int alive = __syncthreads_or(live);
        for (int r_ = r + 1; r_ <= max_r && alive; ++r_) {
            const int d = r_ - r;
            const bool coin_round = (d % P.C) == 0;
            unsigned nv[NJ];
#pragma unroll
            for (int w = 0; w < NJ; w++) nv[w] = 0;
            int decided = -1;
            for (int m0 = 0; m0 < M; m0 += 32) {
                __syncthreads();
                for (int i = tid; i < 32 * NJ; i += blockDim.x) {
                    const int m = m0 + i / NJ;
                    sS[i] = m < M ? P.Sw[((size_t)r_ * M + m) * NJ + (i % NJ)] : 0u;
                }
                if (tid < 32) {
                    const int m = m0 + tid;
                    const int wv = m < M ? P.W[(size_t)r_ * M + m] : -1;
                    vw[tid] = wv >= 0;
                    vcoin[tid] = m < M ? P.coin[(size_t)r_ * M + m] : 0;
                }
                __syncthreads();
                if (tid < 32) {
                    unsigned sw[NJ];
#pragma unroll
                    for (int w = 0; w < NJ; w++) sw[w] = vw[tid] ? sS[tid * NJ + w] : 0u;
                    vsum[tid] = w_wsum<NJ>(sw, unit, stake_s);
                }
                __syncthreads();
                if (live) {
                    unsigned word = 0;
                    for (int b = 0; b < 32 && m0 + b < M; b++) {
                        if (!vw[b]) continue;
                        int vote;
                        if (d == 1) vote = (int)((sS[b * NJ + (mx >> 5)] >> (mx & 31)) & 1);       // swirld.py:256-257
                        else {
                            unsigned an[NJ];
#pragma unroll
                            for (int w = 0; w < NJ; w++) an[w] = sS[b * NJ + w] & pv[w];
                            const i64 yes = w_wsum<NJ>(an, unit, stake_s);                          // majority, :20-27
                            const i64 no = vsum[b] - yes;
                            const int v = no > yes ? 0 : 1;
                            const i64 tt = no > yes ? no : yes;
                            if (!coin_round) {
                                if (3 * tt > P.tot2) { if (decided < 0) decided = v; continue; }    // :261-263
                                vote = v;                                                           // :265
                            } else vote = (3 * tt > P.tot2) ? v : vcoin[b];                         // :267-272
                        }
                        word |= (unsigned)vote << b;
                    }
#pragma unroll
                    for (int w = 0; w < NJ; w++) if (w == (m0 >> 5)) nv[w] = word;
                }
            }
#pragma unroll
            for (int w = 0; w < NJ; w++) pv[w] = nv[w];
            if (live && decided >= 0) {
                P.famous[slot] = (int8_t)decided; P.famous_ev[x] = (int8_t)decided;
                live = false; any_decided = true;
            }
            alive = __syncthreads_or(live);
        }
        const int left = __syncthreads_count(live);
        const int dn = __syncthreads_or(any_decided);
        if (tid == 0) { if (left) atomicAdd(&P.rem[r], left); if (dn) P.done[r] = 1; }
    }
}
template <int NJ, class Src>
__global__ void __launch_bounds__(FW_THREADS) k_w_fame_rounds(Src s) { w_fame_rounds_body<NJ>(params(s)); }

// ------------------------------------------------------------------ find_order (swirld.py:280-311)
// Same plan as swirld_kernels.cuh (A per round, B sequential cuts, C listing, times, sort) with per-round
// arrays of M entries (OrderParams.seg_fw / plan strides are M instead of 64).
#define WPLAN(k) (P.plan + (size_t)(k) * P.plan_stride)

__device__ __forceinline__ void w_order_rounds_body(const OrderParams &P) {
    extern __shared__ int ow_smem[];
    i64 *st = reinterpret_cast<i64 *>(ow_smem);          // [M] stake of fw[i]'s creator
    int *fw = ow_smem + 2 * P.M;                         // [M]
    __shared__ int wtot[32], nf_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, M = P.M, si = blockIdx.x;
    const int r = P.rounds[si];
    int nf_run = 0;
    for (int c0 = 0; c0 < M; c0 += 1024) {               // compaction of the famous witnesses in member order
        const int c = c0 + tid;
        int w = -1, fam = -1;
        if (c < M && r >= 0 && r < P.Rcap) { w = P.W[(size_t)r * M + c]; fam = P.famous[(size_t)r * M + c]; }
        if (w >= 0 && fam < 0) atomicMin(&P.scal[SC_ERR], -3);        // self.famous[w] KeyError, :284
        const bool isf = w >= 0 && fam == 1;
        const unsigned b = __ballot_sync(0xffffffffu, isf);
        if (lane == 0) wtot[warp] = __popc(b);
        __syncthreads();
        int before = nf_run;
        for (int w2 = 0; w2 < warp; w2++) before += wtot[w2];
        if (isf) {
            const int posn = before + __popc(b & ((1u << lane) - 1));
            fw[posn] = w;
            const int cw = P.creator[w];
            st[posn] = P.stake[cw];
            WPLAN(4)[(size_t)si * M + posn] = cw;
        }
        int tot = 0;
        for (int w2 = 0; w2 < 32; w2++) tot += wtot[w2];
        nf_run += tot;
        __syncthreads();
    }
    if (tid == 0) { nf_s = nf_run; P.seg_nf[si] = nf_run; }
    __syncthreads();
    const int nf = nf_s;
    if (tid < 64) {                                      // white = XOR of the famous witnesses' signatures, byte tid
        uint8_t x = 0;
        for (int i = 0; i < nf; i++) x ^= P.sig[(size_t)fw[i] * 64 + tid];
        P.seg_white[(size_t)si * 64 + tid] = x;
    }
    for (int c = tid; c < M; c += 1024) {
        P.seg_fw[(size_t)si * M + c] = c < nf ? fw[c] : -1;
        // reach over all famous witnesses, and the received-threshold: the largest event index v of chain c with
        // more than half the stake of f_w seeing it (:291-293), by bisection (the predicate is monotone in v)
        int U = -1;
        for (int i = 0; i < nf; i++) U = max(U, P.row[(size_t)fw[i] * M + c]);
        int thr = -1;
        if (U >= 0) {
            int lo = 0, hi = U + 1;                      // invariant: f(lo - 1) "true or lo == 0", f(hi) false
            auto f = [&](int v) -> bool {
                i64 acc = 0;
                for (int i = 0; i < nf; i++) if (P.row[(size_t)fw[i] * M + c] >= v) acc += st[i];
                return 2 * acc > P.tot;
            };
            if (f(0)) {
                while (hi - lo > 1) { const int mid = lo + ((hi - lo) >> 1); if (f(mid)) lo = mid; else hi = mid; }
                // lo = largest v with f(v); it is the index of an event some witness shows in column c
                thr = lo;
            }
        }
        WPLAN(0)[(size_t)si * M + c] = thr;
        WPLAN(1)[(size_t)si * M + c] = U;
        WPLAN(2)[(size_t)si * M + c] = thr >= 0 ? P.seq[thr] : -1;
        WPLAN(3)[(size_t)si * M + c] = U >= 0 ? P.seq[U] : -1;
    }
}
template <class Src>
__global__ void __launch_bounds__(1024, 1) k_w_order_rounds(Src s) {
    const OrderParams &P = params(s);
    if constexpr (std::is_pointer<Src>::value) if ((int)blockIdx.x >= P.nrounds) return;
    w_order_rounds_body(P);
}

__device__ __forceinline__ void w_order_cuts_body(const OrderParams &P) {
    extern __shared__ int oc_smem[];
    int *lastord_s = oc_smem, *tbd_s = oc_smem + P.M;
    __shared__ int wtot[32];
    const int c = threadIdx.x, lane = c & 31, warp = c >> 5, M = P.M;
    int lo = c < M ? P.lastord[c] : -1;
    int loseq = lo >= 0 ? P.seq[lo] : -1;
    if (c < M) lastord_s[c] = lo;
    int total = 0;
    __syncthreads();
    for (int si = 0; si < P.nrounds; ++si) {
        const size_t o = (size_t)si * M + (c < M ? c : 0);
        const int thr = WPLAN(0)[o], ua = WPLAN(1)[o], sthr = WPLAN(2)[o], sua = WPLAN(3)[o];
        const int nf = P.seg_nf[si];
        const int fwv = P.seg_fw[o];
        const int cwv = (c < M && fwv >= 0) ? WPLAN(4)[o] : 0;
        const bool ok = c >= nf || fwv > lastord_s[cwv];            // witness slot c is in tbd
        if (c < M) tbd_s[c] = ok ? 1 : 0;
        const int allok = __syncthreads_and(ok);
        int U = ua, sU = sua;
        if (!allok) {
            U = -1;
            for (int i = 0; i < nf; i++)
                if (tbd_s[i] && c < M) U = max(U, P.row[(size_t)P.seg_fw[(size_t)si * M + i] * M + c]);
            sU = U >= 0 ? P.seq[U] : -1;
        }
        const int cut = min(U, thr), scut = U <= thr ? sU : sthr;
        const int cnt = (c < M && cut > lo) ? scut - loseq : 0;
        int inc = cnt;
#pragma unroll
        for (int o2 = 1; o2 < 32; o2 <<= 1) { const int x = __shfl_up_sync(0xffffffffu, inc, o2); if (lane >= o2) inc += x; }
        if (lane == 31) wtot[warp] = inc;
        __syncthreads();
        int before = total, all = 0;
        for (int w2 = 0; w2 < 32; w2++) { if (w2 < warp) before += wtot[w2]; all += wtot[w2]; }
        if (c < M) {
            WPLAN(5)[o] = cnt > 0 ? cut : -1;
            WPLAN(6)[o] = cnt;
            WPLAN(7)[o] = before + inc - cnt;
        }
        if (c == 0) P.seg_start[si] = total;
        total += all;
        if (cnt > 0) { lo = cut; loseq = scut; lastord_s[c] = cut; }
        __syncthreads();
    }
    if (c < M) P.lastord[c] = lo;
    if (c == 0) { P.seg_start[P.nrounds] = total; P.scal[SC_BATCH] = total; }
}
template <class Src> __global__ void __launch_bounds__(1024) k_w_order_cuts(Src s) { w_order_cuts_body(params(s)); }

__device__ __forceinline__ void w_order_list_body(const OrderParams &P) {
    const size_t tot = (size_t)P.nrounds * P.M;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (size_t)gridDim.x * blockDim.x) {
        const int cnt = WPLAN(6)[i];
        if (cnt <= 0) continue;
        int x = WPLAN(5)[i];
        const int off = WPLAN(7)[i], si = (int)(i / P.M);
        for (int j = 0; j < cnt; j++) {
            P.batch_ev[off + j] = x;
            P.batch_seg[off + j] = si;
            x = P.p0[x];
        }
    }
}
template <class Src> __global__ void k_w_order_list(Src s) { w_order_list_body(params(s)); }

__device__ __forceinline__ u64 dbl_key(double d) {       // order-preserving image of a double
    const u64 b = (u64)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double key_dbl(u64 k) {
    const u64 b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)b);
}
// k-th smallest (0-based) of the n keys in shared memory, by one warp: MSB-first radix select
__device__ __forceinline__ u64 warp_select(const u64 *keys, int n, int k, int lane) {
    u64 prefix = 0, mask = 0;
    for (int bit = 63; bit >= 0; bit--) {
        const u64 bm = 1ull << bit;
        int c0 = 0;
        for (int i = lane; i < n; i += 32) { const u64 v = keys[i]; c0 += ((v & mask) == prefix && !(v & bm)) ? 1 : 0; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c0 += __shfl_xor_sync(0xffffffffu, c0, o);
        if (k >= c0) { k -= c0; prefix |= bm; }
        mask |= bm;
    }
    return prefix;
}

#define OW_WARPS 4
__device__ __forceinline__ void w_order_times_body(const OrderParams &P) {
    extern __shared__ u64 ot_smem[];
    const int nbatch = P.scal[SC_BATCH];                 // (left on the device by k_w_order_cuts: no host round trip)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, M = P.M;
    u64 *keys = ot_smem + (size_t)warp * M;
    const int gw = blockIdx.x * OW_WARPS + warp, nw = gridDim.x * OW_WARPS;
    for (int i = gw; i < nbatch; i += nw) {
        const int x = P.batch_ev[i], si = P.batch_seg[i];
        const int c = P.creator[x];
        const int nf = P.seg_nf[si];
        int n = 0;
        __syncwarp();
        for (int k0 = 0; k0 < nf; k0 += 32) {
            const int k = k0 + lane;
            bool sees = false;
            double tv = 0.0;
            if (k < nf) {
                int a = P.seg_fw[(size_t)si * M + k];
                if (P.row[(size_t)a * M + c] >= x) {          // swirld.py:298-302: the event before the first seer (quirk Q10)
                    sees = true;
                    while (P.row[(size_t)a * M + c] >= x && P.p0[a] >= 0) a = P.p0[a];
                    tv = P.t[a];
                }
            }
            const unsigned b = __ballot_sync(0xffffffffu, sees);
            if (sees) keys[n + __popc(b & ((1u << lane) - 1))] = dbl_key(tv);
            n += __popc(b);
        }
        __syncwarp();
        const int ia = n / 2, ib = (n + 1) / 2;
        if (ib >= n) { if (lane == 0) atomicMin(&P.scal[SC_ERR], -2); continue; }   // IndexError, :305
        const u64 ka = warp_select(keys, n, ia, lane);
        const u64 kb = ib == ia ? ka : warp_select(keys, n, ib, lane);
        if (lane == 0) P.ts[i] = __dmul_rn(0.5, __dadd_rn(key_dbl(ka), key_dbl(kb)));
        if (lane < 8) {
            u64 kw = 0;
            for (int b = 0; b < 8; b++)
                kw = (kw << 8) | (u64)(P.seg_white[(size_t)si * 64 + 8 * lane + b] ^ P.sig[(size_t)x * 64 + 8 * lane + b]);
            P.key[(size_t)i * 8 + lane] = kw;
        }
    }
}
template <class Src> __global__ void __launch_bounds__(OW_WARPS * 32) k_w_order_times(Src s) { w_order_times_body(params(s)); }

SW_SRC_INSTANCES(k_w_order_rounds, OrderParams) SW_SRC_INSTANCES(k_w_order_cuts, OrderParams)
SW_SRC_INSTANCES(k_w_order_list, OrderParams) SW_SRC_INSTANCES(k_w_order_times, OrderParams)
SW_SRC_INSTANCES_OF(k_w_fame_rounds, FameParams, 1) SW_SRC_INSTANCES_OF(k_w_fame_rounds, FameParams, 2)
SW_SRC_INSTANCES_OF(k_w_fame_rounds, FameParams, 4) SW_SRC_INSTANCES_OF(k_w_fame_rounds, FameParams, 8)
SW_SRC_INSTANCES_OF(k_w_fame_rounds, FameParams, 16) SW_SRC_INSTANCES_OF(k_w_fame_rounds, FameParams, 32)
