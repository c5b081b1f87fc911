// swirld_kernels.cuh -- hand-written sm_90a kernels of the virtual-voting engine.
//
// Kernel math (fork-free graphs, event id == arrival index, proven against the
// literal oracle by tests/engine_model.py before being written here):
//
//   row(h)[c]  = can_see[h][c]  (swirld.py:72, 203-205, 220)  = max(row(p0)[c], row(p1)[c]),
//                own column := h.  -1 = absent.
//   W[r][c]    = witnesses[r][c] (swirld.py:61, 197, 222), -1 = absent.
//   SM(h)      = { c_ : W[round h][c_] >= 0  and  row(h)[c_] >= W[round h][c_] }   (M-bit mask)
//   T(h)[c_]   = { c  : h sees a round-(round h) event k of member c, and k sees W[round h][c_] }
//              -- the transposed "strongly sees" matrix of swirld.py:207-214.  Inside one
//              round it obeys  T(h) = T(p0) | T(p1) | (SM(h) bit c_) << creator(h), parents of a
//              lower round contribute 0, and a promoted event restarts from its own term.
//   hits[c_]   = stake-weight of (T(p0)[c_] | T(p1)[c_])           (swirld.py:209-214)
//   promoted   = 3 * #{c_ : 3*hits[c_] > 2*tot} > 2*tot            (swirld.py:216, quirk Q3)
//
// All of it is integer / bit work; there is no GEMM here and no tensor-core use.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

typedef unsigned long long u64;
typedef long long i64;

enum { SC_MAX_ROUND = 0, SC_ERR = 1, SC_NEWC = 2, SC_BATCH = 3, SC_NSEG = 4, SC_MAXC = 5, SC_TICKET = 6, SC_COUNT = 8 };

// ---------------------------------------------------------------- small helpers
__device__ __forceinline__ i64 wsum(u64 m, int unit, const i64 *stake_s) {
    if (unit) return (i64)__popcll(m);
    i64 s = 0;
    while (m) {
        int b = __ffsll((long long)m) - 1;
        s += stake_s[b];
        m &= m - 1;
    }
    return s;
}

// ---------------------------------------------------------------- K3-prep: strongly-seen sets
// decide_fame's s(y) (swirld.py:245-254) for every witness y among [first, first+n):
// hits[c_] = sum over members c whose latest seen event k = row(y)[c] has round EXACTLY
// round(y)-1 (quirk Q15) of stake[c] * [c_ in SM(k)];  S[round y][creator y] = {c_ : 3 hits > 2 tot}.
// 32x32 bit-matrix transpose across a warp: lane i gives row i, gets column i (bit b = row b's bit i)
__device__ __forceinline__ unsigned rb_transpose32(unsigned x, int lane) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        const unsigned m0 = s == 16 ? 0x0000ffffu : s == 8 ? 0x00ff00ffu : s == 4 ? 0x0f0f0f0fu : s == 2 ? 0x33333333u : 0x55555555u;
        const unsigned y = __shfl_xor_sync(0xffffffffu, x, s);
        x = (lane & s) ? ((x & ~m0) | ((y & ~m0) >> s)) : ((x & m0) | ((y & m0) << s));
    }
    return x;
}

struct StrongParams {
    int M, first, n, Rcap;
    const int32_t *creator, *row, *round;
    const uint8_t *wit;
    const u64 *SM;
    u64 *S;              // [Rcap][M]
    uint8_t *coin;       // [Rcap][M] coin bit of the witness: sig[0] >> 7 (swirld.py:272)
    const uint8_t *sig;  // [cap][64]
    const i64 *stake;
    i64 tot2;
    int unit;
    const int32_t *list, *list_n;   // optional: the witnesses of the range (else every event of the range is looked at)
    const unsigned *SMw;            // wide path (swirld_wide.cuh): SM as [cap][NJ] words, S as [Rcap][M][NJ] words
    unsigned *Sw;
};

template <int NC>
__global__ void __launch_bounds__(256) k_strong(StrongParams P) {
    const int lane = threadIdx.x & 31;
    const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = gridDim.x * (blockDim.x >> 5);
    const int cnt = P.list ? *P.list_n : P.n;
    const int M = P.M;
    for (int w = gw; w < cnt; w += nw) {
        const int h = P.list ? P.list[w] : P.first + w;
        if (!P.wit[h]) continue;
        const int rh = P.round[h];
        if (rh < 0 || rh >= P.Rcap) continue;
        if (lane == 0) P.coin[(size_t)rh * M + P.creator[h]] = P.sig[(size_t)h * 64] >> 7;
        if (rh < 1) continue;
        const int r = rh - 1;
        u64 mk[NC];
        i64 st[NC], hits[NC];
#pragma unroll
        for (int j = 0; j < NC; j++) {
            const int c = lane + 32 * j;
            mk[j] = 0; st[j] = 0; hits[j] = 0;
            if (c < M) {
                const int k = P.row[(size_t)h * M + c];
                if (k >= 0 && P.round[k] == r) mk[j] = P.SM[k];
                st[j] = P.stake[c];
            }
        }
        __syncwarp();
        // hits[c_] = stake of the members m whose latest seen event (of round r) sees witness c_ of round r:
        // transpose the (member x column) bit matrix in 32x32 blocks, lane c_ then owns its column
#pragma unroll
        for (int jj = 0; jj < NC; jj++)
#pragma unroll
            for (int j = 0; j < NC; j++) {
                const unsigned t = rb_transpose32((unsigned)(mk[jj] >> (32 * j)), lane);   // bit b: member jj*32+b
                if (P.unit) hits[j] += __popc(t);
                else
                    for (int b = 0; b < 32; b++) {
                        const i64 s = __shfl_sync(0xffffffffu, st[jj], b);
                        hits[j] += ((t >> b) & 1) ? s : 0;
                    }
            }
        u64 smask = 0;
#pragma unroll
        for (int j = 0; j < NC; j++)
            smask |= (u64)__ballot_sync(0xffffffffu, 3 * hits[j] > P.tot2) << (32 * j);
        if (lane == 0) P.S[(size_t)rh * M + P.creator[h]] = smask;
    }
}

// ---------------------------------------------------------------- K3: decide_fame
// Every undecided witness x = (r, mx) is an independent recurrence over the voter rounds
// r_ = r+1, r+2, ...: the votes of round r_ on x read only the votes of round r_-1 on x
// (swirld.py:243-272).  So the candidate rounds run side by side, one CTA per round r, four
// threads per witness (each covers a quarter of the <= 64 voters of a round), and a CTA stops as
// soon as all of its witnesses are decided (2-4 voter rounds, unless coin rounds are needed).
// The vote mask of x lives in registers; the voter rows (W, S, coin of round r_) are staged in
// shared memory one round ahead.  Every CTA first finds max_c (swirld.py:226-228); the last CTA to
// finish collects the rounds that reached consensus in ascending order (swirld.py:274-276).  The wide
// kernel (swirld_wide.cuh) adds its tallies up from several CTAs per round, so there k_fame_begin and
// k_fame_finish do these two parts as kernels of their own.
struct FameParams {
    int M, Rcap, C;
    const int32_t *W;        // [Rcap][M]
    const u64 *S;            // [Rcap][M]
    int8_t *famous;          // [Rcap][M]  -1 undecided
    int8_t *famous_ev;       // [cap]
    uint8_t *consensus;      // [Rcap]
    uint8_t *done;           // [Rcap] scratch
    int32_t *rem;            // [Rcap] scratch: undecided witnesses of the round
    const uint8_t *coin;     // [Rcap][M], written by k_strong
    const i64 *stake;
    i64 tot2;
    int unit;
    int32_t *newc;           // [Rcap] out
    int32_t *scal;
    const unsigned *Sw;      // wide path: S as [Rcap][M][NJ] words
};

// max_c: the first round without consensus (swirld.py:226-228), by one whole warp.  Consensus only grows: the scan
// resumes from the last answer.
__device__ __forceinline__ int fame_max_c(const FameParams &P, int lane) {
    int mc = max(P.scal[SC_MAXC], 0);
    for (;;) {
        const int r = mc + lane;
        const bool open = r >= P.Rcap || !P.consensus[r];
        const unsigned b = __ballot_sync(0xffffffffu, open);
        if (b) { mc += __ffs(b) - 1; break; }
        mc += 32;
    }
    return min(mc, P.Rcap);
}

// the rounds of [max_c, max_r] that reached consensus, ascending, into newc (swirld.py:274-276), by one whole CTA
__device__ __forceinline__ void fame_collect(const FameParams &P, int max_c, int max_r) {
    __shared__ int wsum_s[32], s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int r0 = max_c; r0 <= max_r; r0 += blockDim.x) {
        const int r = r0 + tid;
        const bool hit = r <= max_r && __ldcg(P.done + r) && __ldcg(P.rem + r) == 0;
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) wsum_s[warp] = __popc(b);
        __syncthreads();
        int before = s_base;
        for (int w = 0; w < warp; w++) before += wsum_s[w];
        if (hit) { P.newc[before + __popc(b & ((1u << lane) - 1))] = r; P.consensus[r] = 1; }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < nwarp; w++) t += wsum_s[w]; s_base += t; }
        __syncthreads();
    }
    if (tid == 0) { P.scal[SC_NEWC] = s_base; P.scal[SC_MAXC] = max_c; }
}

// The kernels that the sw_batch_* calls launch for several node-views take their parameters from a Src: a value (one
// view per launch) or the device array of the views.  Then blockIdx.y is the view, Pv[blockIdx.y] its parameters,
// staged in shared memory; blockIdx.x and gridDim.x are what they are in a single-view launch, so the grid-stride
// loops, k_fame_rounds' last-CTA ticket and the round kernel's grid barrier count one view's CTAs.  The order grids are
// sized from the view with the most rounds: a CTA beyond its view's rounds exits.
template <typename T>
__device__ __forceinline__ const T &view_params(const T *Pv) {
    __shared__ T Ps;
    static_assert(sizeof(T) % 8 == 0, "staged in 8-byte words");
    for (int i = threadIdx.x; i < (int)(sizeof(T) / 8); i += blockDim.x)     // (a struct copy goes through the stack)
        reinterpret_cast<u64 *>(&Ps)[i] = reinterpret_cast<const u64 *>(Pv + blockIdx.y)[i];
    __syncthreads();
    return Ps;
}
template <typename T>
__device__ __forceinline__ const T &params(const T &P) { return P; }
template <typename T>
__device__ __forceinline__ const T &params(const T *Pv) { return view_params(Pv); }

__device__ __forceinline__ void fame_begin_body(const FameParams &P) {     // one warp
    const int lane = threadIdx.x;
    const int mc = fame_max_c(P, lane);
    if (lane == 0) { P.scal[SC_MAXC] = mc; P.scal[SC_NEWC] = 0; }
    // the open rounds' tallies (the wide kernel adds them up from several CTAs per round)
    const int max_r = P.scal[SC_MAX_ROUND];
    for (int r = mc + lane; r <= max_r && r < P.Rcap; r += 32) { P.rem[r] = 0; P.done[r] = 0; }
}
template <class Src> __global__ void k_fame_begin(Src s) { fame_begin_body(params(s)); }

// M <= 64: each candidate round is one CTA's, which writes its rem / done whole.  (A template over VIEWS so that each
// instance of k_fame_rounds gets its own copy of the body's shared variables and keeps its registers.)
template <bool VIEWS>
__device__ __forceinline__ void fame_rounds_body(const FameParams &P) {
    __shared__ u64 sv[2][64];
    __shared__ i64 vsum[2][64];
    __shared__ i64 stake_s[64];
    __shared__ int vw[2][64];
    __shared__ int vcoin[2][64];
    __shared__ int s_maxc;
    __shared__ bool s_last;
    const int tid = threadIdx.x, M = P.M;
    const int max_r = P.scal[SC_MAX_ROUND];                     // swirld.py:225
    if (tid < 32) { const int mc = fame_max_c(P, tid); if (tid == 0) s_maxc = mc; }
    if (tid < 64) stake_s[tid] = tid < M ? P.stake[tid] : 0;
    __syncthreads();
    const int max_c = s_maxc;
    const int mx = tid >> 2, q = tid & 3, mq0 = q * 16;
    const unsigned qmask = 0xFu << (tid & 28);
    auto load_voters = [&](int r_, int buf) {                   // threads 0..63
        const int w = (tid < M && r_ <= max_r) ? P.W[(size_t)r_ * M + tid] : -1;
        vw[buf][tid] = w;
        const u64 s = w >= 0 ? P.S[(size_t)r_ * M + tid] : 0ull;
        sv[buf][tid] = s;
        vcoin[buf][tid] = (tid < M && r_ <= max_r) ? P.coin[(size_t)r_ * M + tid] : 0;   // swirld.py:272
        vsum[buf][tid] = wsum(s, P.unit, stake_s);
    };
    for (int r = max_c + blockIdx.x; r <= max_r; r += gridDim.x) {   // iter_undetermined, :231-236
        __syncthreads();                                         // (shared buffers of the previous round are free)
        const size_t slot = (size_t)r * M + mx;
        int x = -1;
        bool live = false;
        if (!P.consensus[r] && mx < M) {
            x = P.W[slot];
            live = x >= 0 && P.famous[slot] < 0;
        }
        bool any_decided = false;
        u64 pv = 0;
        if (tid < 64) load_voters(r + 1, (r + 1) & 1);
        int alive = __syncthreads_or(live);
        for (int r_ = r + 1; r_ <= max_r && alive; ++r_) {      // iter_voters, swirld.py:238-241
            const int buf = r_ & 1;
            if (tid < 64) load_voters(r_ + 1, buf ^ 1);         // the next round's voters, one round ahead
            const int d = r_ - r;
            const u64 prev = d > 1 ? pv : 0ull;
            const bool coin_round = (d % P.C) == 0;
            u64 mask = 0;
            int decided = -1;
            if (live) {
                for (int m = mq0; m < mq0 + 16 && m < M; m++) {
                    if (vw[buf][m] < 0) continue;
                    const u64 s = sv[buf][m];
                    int vote;
                    if (d == 1) vote = (int)((s >> mx) & 1);         // swirld.py:256-257
                    else {
                        const i64 yes = wsum(s & prev, P.unit, stake_s);   // majority, :20-27
                        const i64 no = vsum[buf][m] - yes;
                        const int v = no > yes ? 0 : 1;
                        const i64 tt = no > yes ? no : yes;
                        if (!coin_round) {
                            if (3 * tt > P.tot2) { if (decided < 0) decided = v; continue; }  // :261-263
                            vote = v;                                 // :265
                        } else vote = (3 * tt > P.tot2) ? v : vcoin[buf][m];   // :267-272
                    }
                    mask |= (u64)vote << m;
                }
            }
            // combine the four quarters (all deciders agree on the value, see DESIGN.md)
            unsigned mlo = (unsigned)mask, mhi = (unsigned)(mask >> 32);
            mlo |= __shfl_xor_sync(qmask, mlo, 1); mhi |= __shfl_xor_sync(qmask, mhi, 1);
            mlo |= __shfl_xor_sync(qmask, mlo, 2); mhi |= __shfl_xor_sync(qmask, mhi, 2);
            decided = max(decided, __shfl_xor_sync(qmask, decided, 1));
            decided = max(decided, __shfl_xor_sync(qmask, decided, 2));
            pv = ((u64)mhi << 32) | mlo;
            if (live && decided >= 0) {
                if (q == 0) { P.famous[slot] = (int8_t)decided; P.famous_ev[x] = (int8_t)decided; }
                live = false; any_decided = true;
            }
            alive = __syncthreads_or(live);                     // (also: the staged voters are complete)
        }
        const int left = __syncthreads_count(live && q == 0);
        const int dn = __syncthreads_or(any_decided);
        if (tid == 0) { P.rem[r] = left; P.done[r] = dn ? 1 : 0; }
    }
    // the last CTA to get here collects (every CTA read SC_MAXC and the consensus flags before it arrived); the ticket
    // is back at zero for the next call
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        s_last = atomicAdd(reinterpret_cast<unsigned *>(P.scal + SC_TICKET), 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid == 0) P.scal[SC_TICKET] = 0;
    fame_collect(P, max_c, max_r);
}
template <class Src> __global__ void __launch_bounds__(256) k_fame_rounds(Src s) { fame_rounds_body<std::is_pointer<Src>::value>(params(s)); }

template <class Src>
__global__ void __launch_bounds__(1024, 1) k_fame_finish(Src s) {
    const FameParams &P = params(s);
    fame_collect(P, P.scal[SC_MAXC], P.scal[SC_MAX_ROUND]);
}

// ---------------------------------------------------------------- K4: find_order
// One entry of a find_order call's output as the host copies it back behind the scalars: the event, its round received
// (the r of swirld.py:283) and its consensus timestamp (ts[x], swirld.py:305)
struct OrderOut { int32_t ev, rr; double ts; };
static_assert(sizeof(OrderOut) == 4 * sizeof(int32_t), "OrderOut is 4 ints of the scalar block");

struct OrderParams {
    int M, Rcap, nrounds;
    int tx_cap;                  // the order columns: tx[tx_cap] int32, then rounds received int32, then times f64
    const int32_t *rounds;       // [nrounds] sorted(new_c)
    const int32_t *W;
    const int8_t *famous;
    const int32_t *row, *p0, *creator, *seq;
    const double *t;
    const uint8_t *sig;
    const i64 *stake;
    i64 tot;
    int32_t *lastord;            // [M] latest ordered event per member chain, -1 none
    // per-call outputs
    int32_t *batch_ev;           // [cap] events ordered by this call, grouped by segment
    int32_t *batch_seg;          // [cap] segment of each
    int32_t *seg_start;          // [nrounds+1]
    int32_t *seg_fw;             // [nrounds][64] famous witnesses
    int32_t *seg_nf;             // [nrounds]
    uint8_t *seg_white;          // [nrounds][64]
    double *ts;                  // [cap] per batch slot
    u64 *key;                    // [cap][8] big-endian words of white ^ sig
    int32_t *perm;               // [cap] scratch
    int32_t *tx;                 // [cap] transactions (and behind them, see tx_cap, their rounds received and times)
    int32_t *idx;                // [cap]
    int tx_base;
    int out_n;                   // the first out_n events this call orders go behind the scalars (0: the count only)
    int32_t *scal;
    // plan scratch, 8 planes of [plan_stride] ints indexed by segment*64 + chain (or witness slot):
    // 0 thr, 1 reach over all famous witnesses, 2 seq[thr], 3 seq[reach], 4 creator of witness slot, 5 cut, 6 count, 7 offset
    int32_t *plan;
    int plan_stride;
};
// (the batched calls copy it once per view: the new fields sit in what was padding)
static_assert(sizeof(OrderParams) == 232, "OrderParams keeps its size");

// Plan: for each new consensus round the famous witnesses f_w, the whitening
// XOR (swirld.py:284-285) and, per member chain c, the range of events this round
// orders.  On a fork-free graph the reference's BFS over tbd (swirld.py:288-289) reaches
// exactly the not-yet-ordered events x with x <= max_{w in f_w & tbd} row(w)[c], and
// "received" (swirld.py:291-293) is monotone along the chain, so the newly ordered
// events of chain c are (lastord[c], min(reach, received-threshold)].  Only the frontier lastord[]
// carries over from round to round: everything else is computed for all rounds at once (A), a
// 64-thread pass walks the rounds in ascending order (B), the events are listed in parallel (C).
#define PLAN(k) (P.plan + (size_t)(k) * P.plan_stride)

// A: everything about a consensus round that does not depend on what earlier rounds ordered -- one CTA
// per round: famous witnesses, whitening XOR, and per member chain the received-threshold `thr` and the
// reach over ALL famous witnesses (the usual case: none of them is ordered yet).
__device__ __forceinline__ void order_rounds_body(const OrderParams &P) {
    __shared__ int fw[64];
    __shared__ int nf_s;
    __shared__ unsigned ball[2];
    __shared__ int mat[64][64];          // mat[i][c] = row(fw[i])[c]
    __shared__ i64 st[64];               // stake of fw[i]'s creator
    __shared__ int U_s[64], thr_s[64];
    const int tid = threadIdx.x, M = P.M, si = blockIdx.x;
    const int r = P.rounds[si];
    int w = -1, fam = -1;
    if (tid < 64) {
        if (tid < M && r >= 0 && r < P.Rcap) { w = P.W[(size_t)r * M + tid]; fam = P.famous[(size_t)r * M + tid]; }
        if (w >= 0 && fam < 0) atomicMin(&P.scal[SC_ERR], -3);   // self.famous[w] KeyError, :284
        const unsigned b0 = __ballot_sync(0xffffffffu, w >= 0 && fam == 1);
        if ((tid & 31) == 0) ball[tid >> 5] = b0;
        U_s[tid] = -1; thr_s[tid] = -1;
    }
    __syncthreads();
    if (tid < 64) {
        const bool isf = w >= 0 && fam == 1;
        const int pos = (tid >= 32 ? __popc(ball[0]) : 0) + __popc(ball[tid >> 5] & ((1u << (tid & 31)) - 1));
        if (isf) {
            fw[pos] = w;
            const int cw = P.creator[w];
            st[pos] = P.stake[cw];
            PLAN(4)[si * 64 + pos] = cw;
        }
        if (tid == 0) nf_s = __popc(ball[0]) + __popc(ball[1]);
    }
    __syncthreads();
    const int nf = nf_s;
    for (int i = tid; i < nf * 64; i += 1024) {
        const int fi = i >> 6, c = i & 63;
        mat[fi][c] = c < M ? P.row[(size_t)fw[fi] * M + c] : -1;
    }
    if (tid < 64) {   // white = XOR of the famous witnesses' signatures, byte tid
        uint8_t x = 0;
        for (int i = 0; i < nf; i++) x ^= P.sig[(size_t)fw[i] * 64 + tid];
        P.seg_white[(size_t)si * 64 + tid] = x;
        P.seg_fw[(size_t)si * 64 + tid] = tid < nf ? fw[tid] : -1;
        if (tid == 0) P.seg_nf[si] = nf;
    }
    __syncthreads();
    {   // per chain c: reach and received-threshold, 16 thread groups x 64 chains
        const int c = tid & 63, grp = tid >> 6;
        int bestU = -1, bestT = -1;
        for (int i = grp; i < nf; i += 16) {
            const int v = mat[i][c];
            bestU = max(bestU, v);
            if (v > bestT) {     // is v seen by more than half the stake?  (:291-293)
                i64 acc = 0;
                for (int k = 0; k < nf; k++)
                    if (mat[k][c] >= v) acc += st[k];
                if (2 * acc > P.tot) bestT = v;
            }
        }
        if (bestU >= 0) atomicMax(&U_s[c], bestU);
        if (bestT >= 0) atomicMax(&thr_s[c], bestT);
    }
    __syncthreads();
    if (tid < 64) {
        const int thr = thr_s[tid], ua = U_s[tid];
        PLAN(0)[si * 64 + tid] = thr;
        PLAN(1)[si * 64 + tid] = ua;
        PLAN(2)[si * 64 + tid] = thr >= 0 ? P.seq[thr] : -1;
        PLAN(3)[si * 64 + tid] = ua >= 0 ? P.seq[ua] : -1;
    }
}
template <class Src>
__global__ void __launch_bounds__(1024, 1) k_order_rounds(Src s) {
    const OrderParams &P = params(s);
    if constexpr (std::is_pointer<Src>::value) if ((int)blockIdx.x >= P.nrounds) return;
    order_rounds_body(P);
}

// B: the only sequential part -- round after round, what each chain still has to give: the events
// (lastord[c], min(reach, thr)].  A famous witness that an earlier round already ordered does not seed
// the search (swirld.py:288-289, `f_w & tbd`); then the reach is taken over the others.  One thread per
// chain; the next round's vectors are fetched while this one is decided.
__device__ __forceinline__ void order_cuts_body(const OrderParams &P) {
    __shared__ int lastord_s[64], tbd_s[64], wtot[2];
    const int c = threadIdx.x, lane = c & 31, M = P.M;
    int lo = c < M ? P.lastord[c] : -1;
    int loseq = lo >= 0 ? P.seq[lo] : -1;
    lastord_s[c] = lo;
    int total = 0;
    int thr = -1, ua = -1, sthr = -1, sua = -1, fwv = -1, cwv = 0, nf = 0;
    auto fetch = [&](int si, int &thr_, int &ua_, int &sthr_, int &sua_, int &fw_, int &cw_, int &nf_) {
        thr_ = PLAN(0)[si * 64 + c]; ua_ = PLAN(1)[si * 64 + c]; sthr_ = PLAN(2)[si * 64 + c]; sua_ = PLAN(3)[si * 64 + c];
        nf_ = P.seg_nf[si];
        fw_ = P.seg_fw[si * 64 + c];
        cw_ = fw_ >= 0 ? PLAN(4)[si * 64 + c] : 0;
    };
    if (P.nrounds > 0) fetch(0, thr, ua, sthr, sua, fwv, cwv, nf);
    __syncthreads();
    for (int si = 0; si < P.nrounds; ++si) {
        int nthr = -1, nua = -1, nsthr = -1, nsua = -1, nfw = -1, ncw = 0, nnf = 0;
        if (si + 1 < P.nrounds) fetch(si + 1, nthr, nua, nsthr, nsua, nfw, ncw, nnf);
        const bool ok = c >= nf || fwv > lastord_s[cwv];           // witness slot c is in tbd
        tbd_s[c] = ok ? 1 : 0;
        const int allok = __syncthreads_and(ok);
        int U = ua, sU = sua;
        if (!allok) {
            U = -1;
            for (int i = 0; i < nf; i++)
                if (tbd_s[i] && c < M) U = max(U, P.row[(size_t)P.seg_fw[si * 64 + i] * M + c]);
            sU = U >= 0 ? P.seq[U] : -1;
        }
        const int cut = min(U, thr), scut = U <= thr ? sU : sthr;
        const int cnt = (c < M && cut > lo) ? scut - loseq : 0;
        int inc = cnt;                                              // offsets: chains in member order
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
        if (lane == 31) wtot[c >> 5] = inc;
        __syncthreads();
        const int off = total + (c >= 32 ? wtot[0] : 0) + inc - cnt;
        PLAN(5)[si * 64 + c] = cnt > 0 ? cut : -1;
        PLAN(6)[si * 64 + c] = cnt;
        PLAN(7)[si * 64 + c] = off;
        if (c == 0) P.seg_start[si] = total;
        total += wtot[0] + wtot[1];
        if (cnt > 0) { lo = cut; loseq = scut; lastord_s[c] = cut; }
        thr = nthr; ua = nua; sthr = nsthr; sua = nsua; fwv = nfw; cwv = ncw; nf = nnf;
        __syncthreads();
    }
    if (c < M) P.lastord[c] = lo;
    if (c == 0) { P.seg_start[P.nrounds] = total; P.scal[SC_BATCH] = total; }
}
template <class Src> __global__ void __launch_bounds__(64) k_order_cuts(Src s) { order_cuts_body(params(s)); }

// C: list the ordered events of every (round, chain): from the cut down the self-parent chain
__device__ __forceinline__ void order_list_body(const OrderParams &P) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P.nrounds * 64; i += gridDim.x * blockDim.x) {
        const int cnt = PLAN(6)[i];
        if (cnt <= 0) continue;
        int x = PLAN(5)[i];
        const int off = PLAN(7)[i], si = i >> 6;
        for (int j = 0; j < cnt; j++) {
            P.batch_ev[off + j] = x;
            P.batch_seg[off + j] = si;
            x = P.p0[x];
        }
    }
}
template <class Src> __global__ void k_order_list(Src s) { order_list_body(params(s)); }

// Consensus timestamp and sort key of each newly ordered event (swirld.py:295-306):
// one warp per event, lane = famous witness.  For a witness that sees x the reference
// walks down the witness's self-parent chain while the ancestor still sees x
// (:298-302) and takes the timestamp of where it stops (the event before the first
// seer, or the chain root -- quirk Q10); the lopsided median of :305 (quirk Q11).
__device__ __forceinline__ void order_times_body(const OrderParams &P) {
    const int lane = threadIdx.x & 31;
    const int nbatch = P.scal[SC_BATCH];                 // (left on the device by k_order_cuts: no host round trip)
    const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = gridDim.x * (blockDim.x >> 5);
    const int M = P.M;
    for (int i = gw; i < nbatch; i += nw) {
    const int x = P.batch_ev[i], si = P.batch_seg[i];
    const int c = P.creator[x];
    const int nf = P.seg_nf[si];
    double tv[2];
    bool sees[2];
#pragma unroll
    for (int j = 0; j < 2; j++) {
        const int k = lane + 32 * j;
        tv[j] = 0.0; sees[j] = false;
        if (k < nf) {
            int a = P.seg_fw[(size_t)si * 64 + k];
            if (P.row[(size_t)a * M + c] >= x) {
                sees[j] = true;
                while (P.row[(size_t)a * M + c] >= x && P.p0[a] >= 0) a = P.p0[a];
                tv[j] = P.t[a];
            }
        }
    }
    const unsigned b0 = __ballot_sync(0xffffffffu, sees[0]), b1 = __ballot_sync(0xffffffffu, sees[1]);
    const int n = __popc(b0) + __popc(b1);
    // rank of my values among the n times (ties broken by position) -> sorted order
    int rank[2] = {0, 0};
#pragma unroll
    for (int jj = 0; jj < 2; jj++)
        for (int l = 0; l < 32; l++) {
            const double o = __shfl_sync(0xffffffffu, tv[jj], l);
            const bool os = ((jj ? b1 : b0) >> l) & 1;
            if (!os) continue;
            const int opos = jj * 32 + l;
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int mypos = j * 32 + lane;
                if (o < tv[j] || (o == tv[j] && opos < mypos)) rank[j]++;
            }
        }
    const int ia = n / 2, ib = (n + 1) / 2;
    if (ib >= n) { if (lane == 0) atomicMin(&P.scal[SC_ERR], -2); }   // IndexError, :305
    double va = 0.0, vb = 0.0;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        const bool ha = sees[j] && rank[j] == ia, hb = sees[j] && rank[j] == ib;
        const unsigned ma = __ballot_sync(0xffffffffu, ha), mb = __ballot_sync(0xffffffffu, hb);
        if (ma) va = __shfl_sync(0xffffffffu, tv[j], __ffs(ma) - 1);
        if (mb) vb = __shfl_sync(0xffffffffu, tv[j], __ffs(mb) - 1);
    }
    if (lane == 0) P.ts[i] = __dmul_rn(0.5, __dadd_rn(va, vb));
    if (lane < 8) {     // key word `lane` = big-endian bytes 8*lane .. 8*lane+7 of white ^ sig(x)
        u64 kw = 0;
        for (int b = 0; b < 8; b++)
            kw = (kw << 8) | (u64)(P.seg_white[(size_t)si * 64 + 8 * lane + b] ^ P.sig[(size_t)x * 64 + 8 * lane + b]);
        P.key[(size_t)i * 8 + lane] = kw;
    }
    }
}
template <class Src> __global__ void __launch_bounds__(256) k_order_times(Src s) { order_times_body(params(s)); }

__device__ __forceinline__ bool order_less(const OrderParams &P, int a, int b) {
    // a, b are batch slots (-1 = padding = +infinity); (ts, white ^ sig) ascending
    // (swirld.py:306); the slot id is a last resort that never decides on distinct sigs
    if (a < 0) return false;
    if (b < 0) return true;
    const double ta = P.ts[a], tb = P.ts[b];
    if (ta < tb) return true;
    if (ta > tb) return false;
    for (int k = 0; k < 8; k++) {
        const u64 ka = P.key[(size_t)a * 8 + k], kb = P.key[(size_t)b * 8 + k];
        if (ka != kb) return ka < kb;
    }
    return a < b;
}

// One CTA per segment: bitonic sort of the segment's batch slots (padded to a power of
// two with -1 = +infinity; P.perm holds 2 ints per batch slot so the padding is real),
// then append to transactions / idx (swirld.py:306-309), with each event's consensus timestamp and round received at its
// position, and the first out_n of them behind the scalars (OrderOut), where the copy of the scalars brings them back.
__device__ __forceinline__ void order_sort_body(const OrderParams &P) {
    const int si = blockIdx.x;
    const int s0 = P.seg_start[si], cnt = P.seg_start[si + 1] - s0;
    if (cnt <= 0) return;
    const int r = P.rounds[si];
    int n2 = 1;
    while (n2 < cnt) n2 <<= 1;
    int32_t *perm = P.perm + 2 * (size_t)s0;        // n2 < 2 * cnt
    for (int i = threadIdx.x; i < n2; i += blockDim.x) perm[i] = i < cnt ? s0 + i : -1;
    __syncthreads();
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const int a = perm[i], b = perm[l];
                    const bool up = (i & k) == 0;
                    const bool sw = up ? order_less(P, b, a) : order_less(P, a, b);
                    if (sw) { perm[i] = b; perm[l] = a; }
                }
            }
            __syncthreads();
        }
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int b = perm[i], x = P.batch_ev[b], pos = s0 + i;
        const double ts = P.ts[b];
        P.tx[P.tx_base + pos] = x;
        P.tx[(size_t)P.tx_cap + P.tx_base + pos] = r;
        reinterpret_cast<double *>(P.tx + 2 * (size_t)P.tx_cap)[P.tx_base + pos] = ts;
        P.idx[x] = P.tx_base + pos;
        if (pos < P.out_n) { OrderOut &o = reinterpret_cast<OrderOut *>(P.scal + SC_COUNT)[pos]; o.ev = x; o.rr = r; o.ts = ts; }
    }
}
template <class Src>
__global__ void __launch_bounds__(1024, 1) k_order_sort(Src s) {
    const OrderParams &P = params(s);
    if constexpr (std::is_pointer<Src>::value) if ((int)blockIdx.x >= P.nrounds) return;
    order_sort_body(P);
}

// what the host launches: each kernel for one view by value and for the device array of several views
#define SW_SRC_INSTANCES(K, T) template __global__ void K<T>(T); template __global__ void K<const T *>(const T *);
// ... and for a kernel with template parameters before its Src
#define SW_SRC_INSTANCES_OF(K, T, ...) \
    template __global__ void K<__VA_ARGS__, T>(T); template __global__ void K<__VA_ARGS__, const T *>(const T *);
SW_SRC_INSTANCES(k_fame_begin, FameParams) SW_SRC_INSTANCES(k_fame_rounds, FameParams) SW_SRC_INSTANCES(k_fame_finish, FameParams)
SW_SRC_INSTANCES(k_order_rounds, OrderParams) SW_SRC_INSTANCES(k_order_cuts, OrderParams) SW_SRC_INSTANCES(k_order_list, OrderParams)
SW_SRC_INSTANCES(k_order_times, OrderParams) SW_SRC_INSTANCES(k_order_sort, OrderParams)

// what a view's scalar block holds behind the scalars: decide_fame's new rounds (Rcap entries), find_order's output
__device__ __forceinline__ int gather_room(const FameParams &P) { return SC_COUNT + P.Rcap; }
__device__ __forceinline__ int gather_room(const OrderParams &P) { return SC_COUNT + 4 * P.out_n; }

// the first n ints of every view's scalar block (SC_*, and for decide_fame the new rounds or for find_order the output
// behind them) into row v of one staging array: one device-to-host copy brings back what B single calls copy one by one
template <typename T>
__global__ void k_views_gather(const T *Pv, int32_t *out, int n) {
    const T &P = Pv[blockIdx.x];
    const int m = min(n, gather_room(P));
    for (int i = threadIdx.x; i < m; i += blockDim.x) out[(size_t)blockIdx.x * n + i] = P.scal[i];
}

__global__ void k_fill_i32(int32_t *p, int32_t v, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t st = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += st) p[i] = v;
}
