// swirld_rounds.cuh -- round numbers for a chunk of events on the WHOLE GPU
// (Node.divide_rounds, swirld.py:187-222; the can_see rows come from swirld_cansee.cuh).
//
// The reference walks the events one by one because `round[h]` reads `round[parent]`.
// On a fork-free graph the same numbers follow from a monotone predicate instead:
//
//   Wf_r[c]   := member c's FIRST event with round >= r                  (-1: none yet)
//   P_r(h)    := #{c_ : hits_r(h)[c_] > 2T/3} > 2T/3, with
//   hits_r(h)[c_] = sum over members c of stake[c] * [pre(h)[c] >= Wf_r[c] >= 0]
//                                                 * [row(pre(h)[c])[c_] >= Wf_r[c_] >= 0]
//   (pre(h) = can_see row of h with the own column set back to the self-parent, swirld.py:203-205, 220)
//
//   round[h] >= r+1  <=>  P_r(h)          and P_r is monotone along every member's chain.
//
// (=>: an event is promoted from r exactly when the reference's strongly-sees count
// passes, swirld.py:209-219, and every descendant keeps seeing at least as much; <=: P_r(h)
// needs a parent of round >= r.  Using the FIRST event of round >= r instead of the round-r
// witness changes nothing, because seeing a skipping member's event already implies a
// higher round.  tests/test_rounds_model.py keeps the executable proof against the oracle.)
//
// So one cooperative kernel advances all chains round by round.  A step (= one round r):
//   a  every warp computes the masks S_r(k) = {c_ : row(k)[c_] >= Wf_r[c_] >= 0} of up to two events k of
//      the members' ranges [Wf_r[c], end of c's pending window) into the per-event cache `sc`
//      (16-byte entries {mask, mask ^ key(r, launch)}: a stale or torn entry fails the key test);
//   b  one warp per (chain, pending position) tests P_r: it gathers the <= 64 masks of the events its row
//      points at -- polling the entries that are still being produced, there is no barrier between a
//      and b --, transposes the 64x64 bit matrix with warp shuffles and counts its columns; the first
//      hit of a chain is kept by atomicMin;
//   c  ONE grid barrier, then every CTA applies the same bookkeeping: events before the chain's first hit
//      are final at round r, the hit opens round r+1 for the chain (Wf_{r+1}[c]).
// The depth of the computation is the number of ROUNDS in the chunk (~1 per 690 events at 64 members),
// not the number of DAG levels.  An event far ahead of the windows (it sees events whose masks nobody
// prepared) is left untested and truncates its chain's window for this step.
#pragma once
#include "swirld_kernels.cuh"

#define RB_WR 32            // rounds of Wf mirrored in shared memory
#define RB_LMAX 64          // pending events tested per chain and step (at most)
#define RB_THREADS 512       // 16 warps per CTA, one CTA per SM
#define RB_RING 256          // per-member ring of recent events (what precedes the chunk)
#define RB_NPOLL 24          // polls of a mask that is being produced before the reader computes it itself
#define RB_MAXMISS 0         // an event with more unprepared S_r masks than this waits for a later step

struct RbParams {
    int M, first, n, Rcap, L;
    unsigned epoch;             // launch counter (part of the mask-cache key)
    const int32_t *row, *p0, *creator, *seq;
    int32_t *round;             // [cap] out
    int32_t *Wf;                // [Rcap][M] first event of round >= r per member
    ulonglong2 *sc;             // [cap] {S_r(k), S_r(k) ^ key(r)}
    int32_t *cev;               // [cap] chunk events grouped by creator, region [first, first+n)
    int32_t *ccnt, *cmin;       // [MP] per-member count / smallest seq inside the chunk (MP = max(M, 64))
    int32_t *ctot;              // [M] events of the member so far (1 + its largest seq)
    int32_t *gchain;            // [M][RB_RING] the member's most recent events by seq % RB_RING
    int32_t *coff;              // [MP + 1]
    unsigned *bar;              // grid barrier counter of the round kernel (zeroed by k_rb_prep)
    uint8_t *res;               // per-step results of k_rounds_batch, 2 x (64 x u64 + 64 x int)
    const i64 *stake;
    i64 tot2;
    int32_t *scal;
    long long *dbg;             // cycle counters (profiling), may be NULL
    uint8_t *wit;               // [cap]   (finish kernels)
    int32_t *W;                 // [Rcap][M] the reference's witnesses table
    u64 *SM;                    // [cap]
    int32_t *wlist, *wcnt;      // witnesses of the chunk (k_rb_finish -> k_strong)
    const int32_t *cont;        // NULL, or where k_rounds_cluster (swirld_rcluster.cuh) stopped: [0,64) positions, [64,128) rounds,
                                // [128] != 0: there is work left
};

// ---- per-member event lists of the chunk.  Events are divided in arrival order and seq[h] counts the earlier events
// of h's creator, so the per-member counts of a chunk are known on the host (chunk_prep) and arrive by value.
// CM members at most: 64 for the M <= 64 kernels, SW_MAX_MEMBERS (16 KB of parameters) for the any-M kernels.
template <int CM>
struct RbChunk {
    int ccnt[CM];               // events of the member in the chunk
    int cmin[CM];               // the smallest seq among them (0x7f7f7f7f: none)
    int ctot[CM];               // events of the member up to the end of the chunk
    int coff[CM + 1];           // exclusive prefix sum of ccnt
};

// the chunk's meta arrays, cev, and (rsg != NULL, M <= 64) the seq-space rows of swirld_rcluster.cuh in cev order: one
// warp per event
template <int CM>
__global__ void __launch_bounds__(256) k_rb_prep(RbParams P, const __grid_constant__ RbChunk<CM> K, int32_t *rsg) {
    const int tid = threadIdx.x, lane = tid & 31;
    if (blockIdx.x == 0) {
        const int mp = min(CM, max(P.M, 64));                 // (the meta arrays hold max(M, 64) members)
        for (int c = tid; c <= mp; c += blockDim.x) {
            if (c < mp) { P.ccnt[c] = K.ccnt[c]; P.cmin[c] = K.cmin[c]; if (c < P.M) P.ctot[c] = K.ctot[c]; }
            P.coff[c] = K.coff[c];
        }
        if (tid == 0) { *P.bar = 0; *P.wcnt = 0; }
    }
    for (int j = blockIdx.x * 8 + (tid >> 5); j < P.n; j += gridDim.x * 8) {
        const int h = P.first + j, c = P.creator[h];
        const int d = K.coff[c] + P.seq[h] - K.cmin[c];
        if (lane == 0) P.cev[P.first + d] = h;
        if (rsg) {
#pragma unroll
            for (int u = 0; u < 2; u++) {
                const int m = lane + 32 * u;
                const int v = m < P.M ? P.row[(size_t)h * P.M + m] : -1;
                rsg[(size_t)d * 64 + m] = v < 0 ? -1 : P.seq[v];
            }
        }
    }
}

// The rounds run ahead (M <= 64, swirld_b200.cu): after a piece of the round stream, its own ring takes the piece's events
// [rfirst, rfirst + rn), each member's last RB_RING of them (ctot: the members' events up to the piece's end).
struct RbRing {
    int32_t *ring;
    const int32_t *creator, *seq;
    int rfirst, rn;
    int ctot[64];
};

__global__ void __launch_bounds__(256) k_rb_ring(const __grid_constant__ RbRing G) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < G.rn; j += gridDim.x * blockDim.x) {
        const int h = G.rfirst + j, c = G.creator[h], sq = G.seq[h];
        if (G.ctot[c] - sq <= RB_RING) G.ring[c * RB_RING + (sq & (RB_RING - 1))] = h;
    }
}

// ---- after the round kernel, one pass over the chunk: each member's most recent RB_RING events for the next chunk, and
// the reference's witness flags / witnesses table from the finished rounds (swirld.py:221-222, 196-197)
//
// With the rounds run ahead on their own stream (F.on, M <= 64, swirld_b200.cu), the round kernels wrote their own Wf, round
// top and error slot, and this pass publishes what the call's events add to the engine's: the member counts at the call's
// end (F.ctot, also the ring's bound), Wf_r[c] = h for every witness h and r in (round of its self-parent, round h] (the
// entries the round kernel writes: a witness is its member's first event of each round it skips), the round top as the
// largest round, the capacity error when a round reaches Rcap, and any other error the round stream met.
struct RbFold {
    int on;
    int32_t *Wf, *scal, *wnext;   // the engine's Wf and scalars; the witness count of the next call, zeroed here
    const int32_t *rscal;         // the round stream's scalars
    int ctot[64];
};

__global__ void k_rb_finish(RbParams P, const __grid_constant__ RbFold F) {
    if (F.on && blockIdx.x == 0) {
        for (int c = threadIdx.x; c < P.M; c += blockDim.x) P.ctot[c] = F.ctot[c];
        if (threadIdx.x == 0) {
            *F.wnext = 0;
            const int er = F.rscal[SC_ERR];
            if (er < 0 && er != -5) atomicMin(&F.scal[SC_ERR], er);
        }
    }
    int rmax = -1;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < P.n; j += gridDim.x * blockDim.x) {
        const int h = P.first + j, c = P.creator[h], sq = P.seq[h], pa = P.p0[h], r = P.round[h];
        if ((F.on ? F.ctot[c] : P.ctot[c]) - sq <= RB_RING) P.gchain[c * RB_RING + (sq & (RB_RING - 1))] = h;
        const int rp = pa < 0 ? -1 : P.round[pa];
        const bool wit = pa < 0 || r > rp;
        P.wit[h] = wit ? 1 : 0;
        if (wit && r >= 0 && r < P.Rcap) {
            P.W[(size_t)r * P.M + c] = h;
            P.wlist[atomicAdd(P.wcnt, 1)] = h;                // k_strong runs over the witnesses only
        }
        if (F.on && wit)
            for (int q = rp + 1; q <= r && q < P.Rcap; q++) F.Wf[(size_t)q * P.M + c] = h;
        rmax = max(rmax, r);
    }
    if (F.on) {
        for (int o = 16; o > 0; o >>= 1) rmax = max(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
        if ((threadIdx.x & 31) == 0 && rmax >= 0) {
            atomicMax(&F.scal[SC_MAX_ROUND], rmax);
            if (rmax >= P.Rcap) atomicMin(&F.scal[SC_ERR], -5);                   // (the round table is exhausted)
        }
    }
}

// Grid-wide barrier for the co-resident (cooperatively launched) grid.  *ctr is zero at launch and
// counts arrivals for ever; the caller keeps the running target.  The whole of warp 0 polls, so no
// warp leaves the barrier split in two (cooperative_groups' grid.sync() lets thread 0 spin alone and
// its warp then runs every later shuffle on the slow divergent path).
__device__ __forceinline__ void rb_grid_barrier(unsigned *ctr, unsigned &target, unsigned ngrid) {
    __syncthreads();
    target += ngrid;
    if (threadIdx.x < 32) {
        if (threadIdx.x == 0) { __threadfence(); atomicAdd(ctr, 1u); }
        __syncwarp();
        unsigned v;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while ((int)(v - target) < 0);
        __syncwarp();
    }
    __syncthreads();
}

// validity key of a cached mask: the round it was computed for and the launch that computed it (Wf_r can
// gain members between two launches, so a mask of an earlier launch is never reused)
__device__ __forceinline__ u64 rb_key(int r, unsigned epoch) {
    return (u64)(r + 1) * 0x9E3779B97F4A7C15ull ^ (u64)(epoch + 1) * 0xC2B2AE3D27D4EB4Full;
}

// (bx, gx): this CTA's index and the CTA count of ITS hashgraph -- one view's row of the grid (k_rounds_batch)
template <int NC, bool UNIT>
__device__ __forceinline__ void rounds_batch_body(const RbParams &P, const int bx, const int gx) {
    __shared__ int cur[64], pos[64], len[64], off[64];
    __shared__ int Wl[RB_WR][64], Wls[RB_WR][64];             // Wf of the last RB_WR rounds and the chain seq of its entries
    __shared__ i64 stake_s[64];
    __shared__ int s_nfin[64], s_base[64];
    __shared__ int cmin_s[64], ctot_s[64];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int M = P.M, L = P.L;
    const int gw = bx * (blockDim.x >> 5) + warp, nw = gx * (blockDim.x >> 5);
    const i64 thr = P.tot2 / 3;
    const bool lead = bx == 0;
    if (P.cont && __ldcg(P.cont + 128) == 0) return;         // the cluster kernel finished the chunk (the same answer in every CTA)
    // per-step results, double buffered: first hit of a chain as (position << 32 | event), first deferred position
    // (three buffers: the tests of step s+1 start without a grid barrier after the bookkeeping of step s)
    u64 *hitmin = reinterpret_cast<u64 *>(P.res);             // [3][64]
    int *unkmin = reinterpret_cast<int *>(P.res + 3 * 64 * sizeof(u64));   // [3][64]

    int rtop = max(P.scal[SC_MAX_ROUND], 0);
    for (int i = tid; i < RB_WR * 64; i += blockDim.x) {
        const int slot = i >> 6, c = i & 63;
        // the round of (rtop-RB_WR, rtop] that maps to this slot
        const int r = rtop - ((rtop - slot) & (RB_WR - 1));
        const int w = (c < M && r >= 0 && r < P.Rcap) ? __ldcg(P.Wf + (size_t)r * M + c) : -1;
        Wl[slot][c] = w;
        Wls[slot][c] = w >= 0 ? P.seq[w] : 0;
    }
    if (tid < 64) {
        const int c = tid;
        stake_s[c] = c < M ? P.stake[c] : 0;
        int o = 0, l = 0, cu = 0x7fffffff;
        if (c < M) {
            o = P.first + P.coff[c]; l = P.coff[c + 1] - P.coff[c];
            if (l > 0) {
                const int h0 = P.cev[o], pa = P.p0[h0];
                cu = pa < 0 ? 0 : P.round[pa];
            }
        }
        int p = 0;
        if (P.cont && c < M) { p = __ldcg(P.cont + c); cu = __ldcg(P.cont + 64 + c); }
        off[c] = o; len[c] = l; pos[c] = p; cur[c] = cu;
        cmin_s[c] = c < M ? P.cmin[c] : 0; ctot_s[c] = c < M ? P.ctot[c] : 0;
    }
    if (lead && tid < 192) { hitmin[tid] = ~0ull; unkmin[tid] = 0x7fffffff; }
    __syncthreads();
    if (tid < M && len[tid] > 0 && cur[tid] == 0) {          // a member's root opens round 0 for it
        const int h0 = P.cev[off[tid]];
        if (P.p0[h0] < 0) {
            if (rtop < RB_WR) { Wl[0][tid] = h0; Wls[0][tid] = P.seq[h0]; }
            if (lead) P.Wf[tid] = h0;
        }
    }
    unsigned bar_target = 0;
    rb_grid_barrier(P.bar, bar_target, gx);                       // (late roots write the global table only)

    auto in_mirror = [&](int r) -> bool { return r > rtop - RB_WR && r <= rtop; };
    auto wrow = [&](int r, int c) -> int {                    // Wf_r[c]
        if (in_mirror(r)) return Wl[r & (RB_WR - 1)][c];
        return __ldcg(P.Wf + (size_t)r * M + c);
    };

    long long c_miss = 0, tG0 = 0, tG1 = 0, c_g = 0, c_gmax = 0;
    // ---- P_r(h) by one warp; pre = can_see row of h with the own column set back to the self-parent
    auto eval = [&](const int (&pre)[NC], const int (&hi_ev)[NC], int r, bool may_defer) -> int {
        int W[NC];
        bool live[NC];
        u64 m[NC];
        i64 lv = 0;
#pragma unroll
        for (int j = 0; j < NC; j++) {
            const int c = lane + 32 * j;
            W[j] = c < M ? wrow(r, c) : -1;
            live[j] = W[j] >= 0 && pre[j] >= W[j];
            m[j] = 0;
            if (UNIT) lv += __popc(__ballot_sync(0xffffffffu, live[j]));
            else {
                i64 s = live[j] ? stake_s[c] : 0;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                lv += s;
            }
        }
        tG0 = clock64(); tG1 = tG0;
        if (lv <= thr) return 0;                              // hits[c_] <= stake of the live members
        const u64 key = rb_key(r, P.epoch);
        // The masks are produced by other warps in this same step, without a barrier in between: an entry
        // that the producers will write (its event lies inside the member's prepared range) is polled
        // until its key shows up; anything else counts as a miss right away.
        bool valid[NC], expect[NC];
#pragma unroll
        for (int j = 0; j < NC; j++) { valid[j] = !live[j]; expect[j] = live[j] && pre[j] <= hi_ev[j]; }
        for (int poll = 0; poll < RB_NPOLL; poll++) {
#pragma unroll
            for (int j = 0; j < NC; j++)
                if (!valid[j]) {
                    const ulonglong2 e = __ldcg(P.sc + pre[j]);
                    valid[j] = (e.x ^ e.y) == key;
                    m[j] = e.x;
                }
            bool wait = false;
#pragma unroll
            for (int j = 0; j < NC; j++) wait |= expect[j] && !valid[j];
            if (!__any_sync(0xffffffffu, wait)) break;
        }
        __syncwarp();
        {   // an event far ahead of the tested windows sees events nobody prepared: leave it for a later step
            int nm = 0;
#pragma unroll
            for (int j = 0; j < NC; j++) nm += __popc(__ballot_sync(0xffffffffu, live[j] && !valid[j]));
            tG1 = clock64();
            if (may_defer && nm > RB_MAXMISS) return 2;       // (never the chain's first pending event: progress)
        }
#pragma unroll
        for (int jj = 0; jj < NC; jj++) {                     // cache misses: compute S_r(k) together,
            unsigned miss = __ballot_sync(0xffffffffu, live[jj] && !valid[jj]);
            c_miss += __popc(miss);
            while (miss) {                                    // four rows in flight per trip
                int kk[4], ll[4], v[4][NC];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    ll[u] = miss ? __ffs(miss) - 1 : -1;
                    if (miss) miss &= miss - 1;
                    kk[u] = __shfl_sync(0xffffffffu, pre[jj], ll[u] < 0 ? 0 : ll[u]);
#pragma unroll
                    for (int j = 0; j < NC; j++) {
                        const int c = lane + 32 * j;
                        v[u][j] = (ll[u] >= 0 && c < M) ? __ldcg(P.row + (size_t)kk[u] * M + c) : -1;
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (ll[u] < 0) continue;                  // uniform
                    u64 mask = 0;
#pragma unroll
                    for (int j = 0; j < NC; j++)
                        mask |= (u64)__ballot_sync(0xffffffffu, W[j] >= 0 && v[u][j] >= W[j]) << (32 * j);
                    if (lane == 0) P.sc[kk[u]] = make_ulonglong2(mask, mask ^ key);
                    if (lane == ll[u]) m[jj] = mask;
                }
            }
        }
        __syncwarp();                                         // (reconverge: the shuffles below must not take the divergent path)
        // hits[c_] = stake of the live members whose mask has bit c_: transpose the (member x column)
        // bit matrix in 32x32 blocks across the lanes, then lane c_ owns its column as NC words
        unsigned T[NC][NC];                                   // T[jj][j]: bit b = member jj*32+b sees column j*32+lane
#pragma unroll
        for (int jj = 0; jj < NC; jj++) {
            const u64 mine = live[jj] ? m[jj] : 0ull;         // a member that is not live contributes nothing
#pragma unroll
            for (int j = 0; j < NC; j++) T[jj][j] = rb_transpose32((unsigned)(mine >> (32 * j)), lane);
        }
        i64 hits[NC];
#pragma unroll
        for (int j = 0; j < NC; j++) {
            hits[j] = 0;
            if (UNIT) {
#pragma unroll
                for (int jj = 0; jj < NC; jj++) hits[j] += __popc(T[jj][j]);
            } else {
#pragma unroll
                for (int jj = 0; jj < NC; jj++)
#pragma unroll 8
                    for (int b = 0; b < 32; b++) hits[j] += ((T[jj][j] >> b) & 1) ? stake_s[jj * 32 + b] : 0;
            }
        }
        int cnt = 0;
#pragma unroll
        for (int j = 0; j < NC; j++) cnt += __popc(__ballot_sync(0xffffffffu, hits[j] > thr));
        return (i64)cnt > thr ? 1 : 0;
    };

    long long c_t[6] = {0, 0, 0, 0, 0, 0}, c_nev = 0, c_steps = 0, c_maxev = 0, c_sumev = 0, c_def = 0;
    for (int step = 0;; ++step) {
        const long long t0 = clock64();
        // ---- lowest open round (every warp for itself: the chain state is identical in all CTAs)
        int rmin = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int c = lane + 32 * j;
            if (c < M && pos[c] < len[c]) rmin = min(rmin, cur[c]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) rmin = min(rmin, __shfl_xor_sync(0xffffffffu, rmin, o));
        if (rmin == 0x7fffffff) break;                        // every chain is done
        const int buf = step % 3;
        // ---- this warp's test of the step: fetch its inputs now, they are needed after the barrier
        const int tc = gw / L, tj = gw - tc * L;              // one (chain, position) per warp (the whole GPU on one view: M * L <= nw)
        const bool act = tc < M && pos[tc] < len[tc] && cur[tc] == rmin && pos[tc] + tj < len[tc];
        int th = -1, tpa = -1, tpre[NC];
        if (act) th = P.cev[off[tc] + pos[tc] + tj];          // (its dependent loads are issued after the range arithmetic)
        // ---- S_rmin(k) of every event the tests can meet: per member, its events from Wf_rmin[c] up to
        //      the end of its pending window (one warp per event, all SMs).  Ranges in registers:
        //      lane holds members lane and lane+32.
        int rlo[2], rcnt[2], rinc[2], rhi[2];
        const bool mir = in_mirror(rmin);
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int c = lane + 32 * j;
            int lo = 0, cnt = 0;
            if (c < M) {
                const int w = wrow(rmin, c);
                if (w >= 0) {
                    lo = mir ? Wls[rmin & (RB_WR - 1)][c] : __ldcg(P.seq + w);
                    const int hi = len[c] > 0 ? cmin_s[c] + min(len[c], pos[c] + L) : ctot_s[c];
                    cnt = max(0, min(hi - lo, RB_RING));
                }
            }
            rlo[j] = lo; rcnt[j] = cnt;
            // the last event of the prepared range, as an event index (what a test compares its pre[] with)
            int hv = -1;
            if (cnt > 0) {
                const int sq = lo + cnt - 1;
                if (len[c] > 0 && sq >= cmin_s[c]) hv = P.cev[off[c] + sq - cmin_s[c]];
                else {
                    const int before = len[c] > 0 ? cmin_s[c] : ctot_s[c];
                    hv = (before - sq <= RB_RING) ? __ldcg(P.gchain + c * RB_RING + (sq & (RB_RING - 1))) : -1;
                }
            }
            rhi[j] = hv;
            int inc = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
            rinc[j] = inc;
        }
        const int totA = __shfl_sync(0xffffffffu, rinc[0], 31);
        rinc[1] += totA;
        const int total = __shfl_sync(0xffffffffu, rinc[1], 31);
        if (act) {
            tpa = P.p0[th];
#pragma unroll
            for (int j = 0; j < NC; j++) {
                const int c = lane + 32 * j;
                tpre[j] = c < M ? __ldcg(P.row + (size_t)th * M + c) : -1;
            }
        }
        const long long tA0 = clock64();
        {
            const u64 key = rb_key(rmin, P.epoch);
            // candidate i -> its event (the member whose range holds i is the first with inclusive prefix > i)
            auto candidate = [&](int i) -> int {
                if (i >= total) return -1;
                int c, base, lo;
                if (i < totA) {
                    c = __popc(__ballot_sync(0xffffffffu, rinc[0] <= i));
                    base = __shfl_sync(0xffffffffu, rinc[0] - rcnt[0], c); lo = __shfl_sync(0xffffffffu, rlo[0], c);
                } else {
                    const int l = __popc(__ballot_sync(0xffffffffu, rinc[1] <= i));
                    c = 32 + l;
                    base = __shfl_sync(0xffffffffu, rinc[1] - rcnt[1], l); lo = __shfl_sync(0xffffffffu, rlo[1], l);
                }
                const int sq = lo + (i - base);
                if (len[c] > 0 && sq >= cmin_s[c]) return P.cev[off[c] + sq - cmin_s[c]];
                // before the chunk: the ring holds the member's last RB_RING events of the earlier chunks
                const int before = len[c] > 0 ? cmin_s[c] : ctot_s[c];
                return (before - sq <= RB_RING) ? __ldcg(P.gchain + c * RB_RING + (sq & (RB_RING - 1))) : -1;
            };
            for (int i = gw; i < total; i += 2 * nw) {       // two rows in flight per trip
                const int k0 = candidate(i), k1 = candidate(i + nw);
                int v0[NC], v1[NC], wv[NC];
#pragma unroll
                for (int j = 0; j < NC; j++) {
                    const int cc = lane + 32 * j;
                    wv[j] = cc < M ? wrow(rmin, cc) : -1;
                    v0[j] = (k0 >= 0 && cc < M) ? __ldcg(P.row + (size_t)k0 * M + cc) : -1;
                    v1[j] = (k1 >= 0 && cc < M) ? __ldcg(P.row + (size_t)k1 * M + cc) : -1;
                }
                u64 mask0 = 0, mask1 = 0;
#pragma unroll
                for (int j = 0; j < NC; j++) {
                    mask0 |= (u64)__ballot_sync(0xffffffffu, wv[j] >= 0 && v0[j] >= wv[j]) << (32 * j);
                    mask1 |= (u64)__ballot_sync(0xffffffffu, wv[j] >= 0 && v1[j] >= wv[j]) << (32 * j);
                }
                if (lane == 0 && k0 >= 0) P.sc[k0] = make_ulonglong2(mask0, mask0 ^ key);
                if (lane == 0 && k1 >= 0) P.sc[k1] = make_ulonglong2(mask1, mask1 ^ key);
            }
        }
        const long long tA1 = clock64();
        const long long tS1 = tA1;
        // ---- test the pending windows
        if (act) {
            int hit = 0;
            if (tpa >= 0) {
#pragma unroll
                for (int j = 0; j < NC; j++) if (lane + 32 * j == tc) tpre[j] = tpa;
                int thi[NC];
#pragma unroll
                for (int j = 0; j < NC; j++) thi[j] = rhi[j];
                hit = eval(tpre, thi, rmin, tj > 0);
            }
            if (lane == 0) {
                if (hit == 1) atomicMin(hitmin + buf * 64 + tc, ((u64)tj << 32) | (unsigned)th);
                if (hit == 2) atomicMin(unkmin + buf * 64 + tc, tj);
            }
            const long long e1 = clock64() - tS1;
            c_maxev = e1 > c_maxev ? e1 : c_maxev; c_sumev += e1; c_nev++; c_def += hit == 2;
            c_g += tG1 - tG0; c_gmax = max(c_gmax, tG1 - tG0);
        }
        // a view that shares the launch with others has fewer warps than (chain, position) pairs: the rest of its tests, in turn
        for (int item = gw + nw; item < M * L; item += nw) {
            const int c2 = item / L, j2 = item - c2 * L;
            if (!(pos[c2] < len[c2] && cur[c2] == rmin && pos[c2] + j2 < len[c2])) continue;
            const int h2 = P.cev[off[c2] + pos[c2] + j2], pa2 = P.p0[h2];
            int hit = 0;
            if (pa2 >= 0) {
                int pre2[NC], thi[NC];
#pragma unroll
                for (int j = 0; j < NC; j++) {
                    const int c = lane + 32 * j;
                    pre2[j] = c < M ? __ldcg(P.row + (size_t)h2 * M + c) : -1;
                    if (c == c2) pre2[j] = pa2;
                    thi[j] = rhi[j];
                }
                hit = eval(pre2, thi, rmin, j2 > 0);
            }
            if (lane == 0) {
                if (hit == 1) atomicMin(hitmin + buf * 64 + c2, ((u64)j2 << 32) | (unsigned)h2);
                if (hit == 2) atomicMin(unkmin + buf * 64 + c2, j2);
            }
        }
        // the rows the next steps will read first (masks and tests of the events just beyond the windows):
        // pull them into L2 now, off the critical path
        if (tc < M && lane < NC * 2) {
            const int idx = pos[tc] + L + tj;
            if (idx < len[tc]) {
                const int h = P.cev[off[tc] + idx];
                const char *ptr = reinterpret_cast<const char *>(P.row + (size_t)h * M) + lane * 128;
                if (lane * 128 < M * 4) asm volatile("prefetch.global.L2 [%0];" :: "l"(ptr));
            }
        }
        const long long t1 = clock64();
        rb_grid_barrier(P.bar, bar_target, gx);
        const long long t2 = clock64();
        // ---- identical bookkeeping in every CTA (only CTA 0 writes the global tables)
        int ft = -1, win = 0, hnew = -1;
        bool mine = false;
        if (tid < M && pos[tid] < len[tid] && cur[tid] == rmin) {
            mine = true;
            win = min(L, len[tid] - pos[tid]);
            const u64 hm = __ldcg(hitmin + buf * 64 + tid);
            const int unk = min(__ldcg(unkmin + buf * 64 + tid), win);   // first position left untested
            if (hm != ~0ull) { ft = (int)(hm >> 32); hnew = (int)(unsigned)hm; }
            if (ft >= 0 && unk < ft) ft = -1;                  // an untested event precedes the first hit
            if (ft < 0) win = unk;                             // only the tested prefix is final
        }
        if (__syncthreads_or(mine && ft >= 0 && rmin + 1 > rtop)) {   // open the shared-memory row of round rmin+1
            rtop = rmin + 1;
            if (tid < 64) { Wl[rtop & (RB_WR - 1)][tid] = -1; Wls[rtop & (RB_WR - 1)][tid] = 0; }
            if (rtop >= P.Rcap && tid == 0 && lead) atomicMin(&P.scal[SC_ERR], -5);
            __syncthreads();
        }
        if (tid < 64) {
            int nfinal = 0, o = 0;
            if (mine) {
                const int c = tid;
                o = off[c] + pos[c];
                nfinal = ft >= 0 ? ft : win;
                if (ft >= 0) {
                    cur[c] = rmin + 1;
                    if (rmin + 1 < P.Rcap) {
                        Wl[(rmin + 1) & (RB_WR - 1)][c] = hnew;
                        Wls[(rmin + 1) & (RB_WR - 1)][c] = cmin_s[c] + pos[c] + ft;
                        if (lead) P.Wf[(size_t)(rmin + 1) * M + c] = hnew;
                    }
                }
                pos[c] += nfinal;
            }
            s_nfin[tid] = nfinal; s_base[tid] = o;
            if (lead) { const int nb2 = (buf + 2) % 3; hitmin[nb2 * 64 + tid] = ~0ull; unkmin[nb2 * 64 + tid] = 0x7fffffff; }
        }
        __syncthreads();
        // final rounds of the events before the first hit, spread over the CTAs
        for (int i = bx + gx * tid; i < M * RB_LMAX; i += gx * blockDim.x) {
            const int c = i / RB_LMAX, j = i % RB_LMAX;
            if (j < s_nfin[c]) P.round[P.cev[s_base[c] + j]] = rmin;
        }
        const long long t3 = clock64();
        c_t[0] += tA0 - t0; c_t[1] += tA1 - tA0; c_t[2] += tS1 - tA1; c_t[3] += t1 - tS1; c_t[4] += t2 - t1; c_t[5] += t3 - t2;
        c_steps++;
    }
    if (P.dbg && lane == 0) {
        atomicMax((unsigned long long *)P.dbg + 8, (unsigned long long)c_maxev);
        atomicAdd((unsigned long long *)P.dbg + 9, (unsigned long long)c_miss);
        atomicAdd((unsigned long long *)P.dbg + 10, (unsigned long long)c_sumev);
        atomicAdd((unsigned long long *)P.dbg + 11, (unsigned long long)c_nev);
        atomicAdd((unsigned long long *)P.dbg + 12, (unsigned long long)c_def);
        atomicAdd((unsigned long long *)P.dbg + 13, (unsigned long long)c_g);
        atomicMax((unsigned long long *)P.dbg + 14, (unsigned long long)c_gmax);
    }
    if (P.dbg && lane == 0 && warp == 0 && bx == 0) {
        unsigned long long *o = (unsigned long long *)P.dbg;
        for (int i = 0; i < 6; i++) atomicAdd(&o[i], (unsigned long long)c_t[i]);
        atomicAdd(&o[6], (unsigned long long)c_steps);
    }
    if (lead && tid == 0 && P.n > 0) P.scal[SC_MAX_ROUND] = rtop;
}

// Several independent node-views (SURVEY.md section 8f-3: the simulation's M nodes each recompute consensus on nearly
// the same graph, swirld.py:331-345) go in ONE cooperative launch: view blockIdx.y runs on its own row of CTAs with its
// own parameters, barrier counter and result buffers.  The path is latency-bound (one grid-wide step per round), so
// small CTA groups advancing side by side use the GPU far better than one view on all of it.
template <int NC, bool UNIT, class Src>
__global__ void __launch_bounds__(RB_THREADS, 1) k_rounds_batch(Src s) {
    rounds_batch_body<NC, UNIT>(params(s), blockIdx.x, gridDim.x);
}
SW_SRC_INSTANCES_OF(k_rounds_batch, RbParams, 1, false) SW_SRC_INSTANCES_OF(k_rounds_batch, RbParams, 1, true)
SW_SRC_INSTANCES_OF(k_rounds_batch, RbParams, 2, false) SW_SRC_INSTANCES_OF(k_rounds_batch, RbParams, 2, true)

// ---- SM(h) = {c_ : W[round h][c_] >= 0 and row(h)[c_] >= W[round h][c_]}, one warp per event
template <int NC>
__global__ void __launch_bounds__(256) k_rb_seenmask(RbParams P) {
    const int lane = threadIdx.x & 31;
    const int j0 = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (j0 >= P.n) return;
    const int h = P.first + j0, r = P.round[h], M = P.M;
    u64 mask = 0;
#pragma unroll
    for (int j = 0; j < NC; j++) {
        const int c = lane + 32 * j;
        int w = -1, v = -1;
        if (c < M && r >= 0 && r < P.Rcap) { w = P.W[(size_t)r * M + c]; v = P.row[(size_t)h * M + c]; }
        mask |= (u64)__ballot_sync(0xffffffffu, w >= 0 && v >= w) << (32 * j);
    }
    if (lane == 0) P.SM[h] = mask;
}
