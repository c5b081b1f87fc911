// swirld_rcluster.cuh -- the round numbers of a chunk (Node.divide_rounds, swirld.py:187-222) inside ONE thread-block
// cluster, M <= 64.
//
// swirld_rounds.cuh advances all member chains one round per grid-wide step; a step there is ~8 dependent trips
// through L2 (rows, mask cache, atomics, the grid barrier, the results): 6 us, 1461 times per million events.  The
// work of a step is small (a few thousand masks and tests), so this kernel keeps everything a step touches in the
// shared memory of 16 CTAs and moves it over distributed shared memory (~200 cycles a hop):
//
//   * rows in SEQ space: rs(h)[c] = the chain position (swirld.py's implicit per-creator sequence number) of the
//     event of member c that h sees (k_rb_prep, from the can_see table).  Every comparison of the scheme
//     ("row(k)[c_] >= Wf_r[c_]") holds in seq space as it does in index space -- a member's events are ordered the
//     same way in both -- and a mask S_r(k) is addressed by (member, position) without any lookup.
//   * CTA q owns chains 4q..4q+3: a window of RC_WN consecutive rows per chain (and their event indices) in its
//     shared memory, filled one step ahead by bulk copies (one or two per chain and step, counted on an mbarrier;
//     the rows' event indices by cp.async).  The state of chain c (position, round, window bounds) lives
//     in the registers of thread c of EVERY CTA: all 16 CTAs do the same bookkeeping from the same results, so no
//     decision ever has to be communicated.
//   * a step (round r = lowest open round):
//       a  the owner computes S_r of its members' events [Wls_r[m], mend[m]) from its window into its own mask table
//          and sends each member's masks to the other 15 tables as 16-byte st.async stores, which count their bytes
//          on an mbarrier of the receiver (the receiver knows how many bytes to expect: it does the same arithmetic);
//       b  the owner finds each chain's first pending event that passes P_r (1) or sees beyond the prepared masks (2):
//          unit stake: all 32 positions of the window at once, 8 tests per warp, 4 lanes x 16 members per test --
//          a lane adds the masks of its live members into a bit-sliced (vertical) counter with carry-save adders,
//          the 4 lanes add their counters by shuffles, and the 64 column counts are compared with the threshold
//          plane by plane; what needs only the CTA's own rows runs before the wait for the others' masks.
//          Integer stakes: a 5-ary search with the chain's 4 warps (P_r and "beyond the masks" are monotone along
//          a chain), one test of swirld_rounds.cuh's kind per warp and pass;
//       c  (first position, kind) of every chain to every CTA, again by st.async + mbarrier;
//       d  identical bookkeeping in every CTA; the owner stores the final rounds and Wf, the window slides.
//     (Plain DSMEM stores and barrier.cluster instead of st.async + mbarrier are slower: the release fence of the
//     barrier also waits for the step's global stores.)
//   * whatever the windows cannot decide -- no progress for RC_STALL steps, a chain more than RB_WR rounds behind,
//     rows further before the chunk than RC_REACH -- hands the REST of the chunk to k_rounds_batch through `cont`
//     (positions and rounds per chain).  tests/test_rounds_cluster_model.py is the executable model.
#pragma once
#include "swirld_rounds.cuh"

#define RC_CS 16            // CTAs per cluster
#define RC_CPC 4            // chains per CTA
#define RC_WPC 4            // warps per chain
#define RC_THREADS 512
#define RC_LW 32            // pending events searched per chain and step
#define RC_WN 128           // rows per chain in shared memory (power of two)
#define RC_MR 64            // masks per member and step
#define RC_MRS 66           // ... and the stride of a member's masks in the table: rows 4 banks apart, 16-byte aligned
#define RC_PF 32            // rows loaded beyond the searched window
#define RC_PASSES 3         // (RC_WPC + 1) ^ RC_PASSES >= RC_LW + 1
#define RC_STALL 3
#define RC_REACH (RC_WN / 2) // rows before the chunk that a launch may need (from the ring)
#define RC_INF 0x7fffffff
#define RC_BIG 0x3fffffff    // "no event of this round": above every chain position

struct RcParams {
    RbParams R;
    const int32_t *rsg;      // [n][64] seq-space rows of the chunk's events in cev order (k_rb_prep)
    int32_t *cont;           // [0,64) positions, [64,128) rounds, [128] 1 = k_rounds_batch has work left
    unsigned *slog;          // per-CTA step log (profiling, k_rounds_cluster_log), NULL unless the engine was created with SW_RC_STEPS
};

// The step log: a header of RC_LOGH words ([0] steps logged by the launches so far, [1] capacity in steps), then one
// record of RC_NLOG words per (step, CTA), in cycles of that CTA's thread 0.  Clocks of different SMs are not
// comparable, but every CTA starts a step when the same result words arrive and tests when the same masks arrive, so
// RL_SENDER (results in -> own masks pushed) and RL_TESTER (masks in -> own results sent) can be compared across the
// CTAs of one step: the largest of each is the CTA the others wait for.  tools/rc_steps.py reads it.
#define RC_LOGH 16
#define RC_NLOG 16
enum {
    RL_WAIT,    // wait for the last step's results
    RL_CTL,     // bookkeeping (warp 0) and the wait for the rows issued a step ago
    RL_BAR1,    // block barrier after the bookkeeping
    RL_MASK,    // masks of my members into my table
    RL_BAR2,    // block barrier before the push
    RL_PUSH,    // my members' masks to the 15 other tables
    RL_TEST1,   // test phase 1 (my rows only)
    RL_MWAIT,   // wait for the other CTAs' masks
    RL_TEST2,   // test phase 2 (the masks)
    RL_BAR3,    // block barrier after the tests
    RL_SEND,    // results of my chains to every CTA
    RL_DEFER,   // final rounds of the last step, the copies of the next rows
    RL_SENDER,  // results in -> masks pushed
    RL_TESTER,  // masks in -> results sent
};

#define RC_SMEM_ROWS ((size_t)RC_CPC * RC_WN * 64 * 4)
#define RC_SMEM_MASK ((size_t)2 * 64 * RC_MRS * 8)   // two mask tables: a CTA may receive the next step's masks while it still tests
#define RC_SMEM_WLS ((size_t)RB_WR * 64 * 4)
#define RC_SMEM_BYTES (RC_SMEM_ROWS + RC_SMEM_MASK + RC_SMEM_WLS + 512 + 10240)

__device__ __forceinline__ unsigned rc_cta_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void rc_cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void rc_cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void rc_cluster_sync() { rc_cluster_arrive(); rc_cluster_wait(); }
__device__ __forceinline__ unsigned rc_map(const void *p, unsigned rank) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
    return r;
}
// one bulk copy (the TMA unit) of `bytes` (a multiple of 16, both addresses 16-byte aligned) from global memory into my
// shared memory, counted on the mbarrier `mbar` of my CTA
__device__ __forceinline__ void rc_bulk(void *dst, const void *src, unsigned bytes, unsigned mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}

__device__ __forceinline__ void rc_cp4(void *dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
// carry-save adder over 64 bit columns: a + b + c = 2 * h + l
__device__ __forceinline__ void rc_csa(u64 &h, u64 &l, u64 a, u64 b, u64 c) {
    const u64 u = a ^ b;
    h = (a & b) | (u & c);
    l = u ^ c;
}
// bit-sliced a[0..NB) += the same number of the lane `delta` away; the sum has NB + 1 bits
template <int NB>
__device__ __forceinline__ void rc_vadd_xor(u64 (&a)[8], int delta) {
    u64 carry = 0;
#pragma unroll
    for (int k = 0; k < NB; k++) {
        const u64 b = __shfl_xor_sync(0xffffffffu, a[k], delta);
        u64 h, l;
        rc_csa(h, l, a[k], b, carry);
        a[k] = l; carry = h;
    }
    a[NB] = carry;
}

// ---- message passing without fences: st.async delivers the data AND counts its bytes on an mbarrier of the receiving CTA
__device__ __forceinline__ void rc_mbar_init(unsigned mbar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(mbar), "r"(count) : "memory"); }
__device__ __forceinline__ void rc_mbar_expect(unsigned mbar, unsigned bytes) {
    asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }" :: "r"(mbar), "r"(bytes) : "memory");
}
// false: the bytes did not arrive within ~2 s (a bug or a dead peer CTA; the caller gives up instead of hanging the GPU).
// Generous on purpose: under compute-sanitizer a peer CTA can be three orders of magnitude slower than usual.
__device__ __forceinline__ bool rc_mbar_wait(unsigned mbar, unsigned parity) {
    const long long t0 = clock64();
    for (;;) {
        unsigned ok;
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(mbar), "r"(parity) : "memory");
        if (ok) return true;
        if (clock64() - t0 > 4000000000ll) return false;
    }
}
__device__ __forceinline__ void rc_sta_v4(unsigned addr, uint4 v, unsigned mbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
                 :: "r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(mbar) : "memory");
}
__device__ __forceinline__ void rc_sta_u32(unsigned addr, unsigned v, unsigned mbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" :: "r"(addr), "r"(v), "r"(mbar) : "memory");
}

template <bool UNIT, bool LOG>
__device__ __forceinline__ void rounds_cluster_body(const RcParams &Q) {
    const RbParams &P = Q.R;
    extern __shared__ __align__(16) unsigned char rc_smem[];
    int (*rsw)[RC_WN][64] = reinterpret_cast<int (*)[RC_WN][64]>(rc_smem);                       // [chain][slot][member]
    u64 (*maskbuf0)[RC_MRS] = reinterpret_cast<u64 (*)[RC_MRS]>(rc_smem + RC_SMEM_ROWS);           // [2][member][offset]
    int (*Wls)[64] = reinterpret_cast<int (*)[64]>(rc_smem + RC_SMEM_ROWS + RC_SMEM_MASK);       // seq of Wf_r[c], -1: none
    i64 *stake_s = reinterpret_cast<i64 *>(rc_smem + RC_SMEM_ROWS + RC_SMEM_MASK + RC_SMEM_WLS);
    int *iv = reinterpret_cast<int *>(stake_s + 64);
    // what the chain threads (tid < 64, one per member chain) publish for the other warps, per step
    int *slo = iv, *smend = iv + 64, *swin = iv + 128, *spos = iv + 192, *s_old = iv + 256, *wldp = iv + 320;
    int *s_nfin = iv + 384, *s_base = iv + 448, *xres = iv + 512, *wp = iv + 576, *cnts = iv + 640;
    // constants of the launch
    int *off = iv + 704, *cmin_s = iv + 768, *coff_s = iv + 832, *len_s = iv + 896, *ctot_s = iv + 960, *cur0 = iv + 1024;
    int *ws = iv + 1088;                                                                         // [8] warp results
    int *sa = iv + 1096, *sb = sa + RC_CPC, *svb = sb + RC_CPC, *tres = svb + RC_CPC;             // tres[RC_CPC][RC_WPC]
    int (*cevw)[RC_WN] = reinterpret_cast<int (*)[RC_WN]>(iv + 1152);                           // event index of every window row
    int *vres = iv + 1152 + RC_CPC * RC_WN;                                                      // [RC_CPC][RC_LW] test results
    int2 (*cst)[64] = reinterpret_cast<int2 (*)[64]>(iv + 1792);                                 // [chain][member] {threshold, span}
    const unsigned mbar0 = (unsigned)__cvta_generic_to_shared(iv + 2304);                        // mbarriers: masks (2 tables), results
    unsigned *tsm = reinterpret_cast<unsigned *>(iv + 2320);     // step log, thread 0: [0, 15) clocks, [16] first record, [17] capacity

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int M = P.M;
    const int bx = (int)rc_cta_rank();
    const bool lead = bx == 0;
    const i64 thr = P.tot2 / 3;

    int rtop = max(P.scal[SC_MAX_ROUND], 0);
    for (int i = tid; i < RB_WR * 64; i += RC_THREADS) {
        const int slot = i >> 6, c = i & 63;
        const int r = rtop - ((rtop - slot) & (RB_WR - 1));
        const int w = (c < M && r >= 0 && r < P.Rcap) ? __ldcg(P.Wf + (size_t)r * M + c) : -1;
        Wls[slot][c] = w >= 0 ? P.seq[w] : -1;
    }
    // ---- the launch-time state of chain c, by thread c
    int my_cur = RC_INF, my_len = 0, my_cmin = 0, my_ctot = 0, my_wlo = 0, my_wld = 0, my_wrd = 0;
    if (tid < 64) {
        const int c = tid;
        stake_s[c] = c < M ? P.stake[c] : 0;
        int o = 0, co = 0;
        bool root = false;
        if (c < M) {
            co = P.coff[c]; o = P.first + co; my_len = P.coff[c + 1] - co;
            my_ctot = P.ctot[c];
            if (my_len > 0) {
                const int h0 = P.cev[o], pa = P.p0[h0];
                my_cur = pa < 0 ? 0 : P.round[pa];
                my_cmin = P.cmin[c];
                root = pa < 0;
                if (root && lead) P.Wf[c] = h0;                 // a member's root opens round 0 for it
            }
        }
        off[c] = o; coff_s[c] = co; cmin_s[c] = my_cmin; len_s[c] = my_len; ctot_s[c] = my_ctot; cur0[c] = my_cur;
        xres[c] = root ? 1 : 0;
    }
    __syncthreads();
    if (tid < 64 && xres[tid] && rtop < RB_WR) Wls[0][tid] = 0;
    __syncthreads();

    if (tid == 0) {
        rc_mbar_init(mbar0, 1); rc_mbar_init(mbar0 + 8, 1); rc_mbar_init(mbar0 + 16, 1);
        rc_mbar_init(mbar0 + 24, RC_CPC);                       // the window rows of my chains: one arrival per chain and step
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    int handed = 0;
    // ---- the windows at launch: [wlo, wld) from the chunk's seq rows, what precedes the chunk through the ring
    {
        int r0 = RC_INF;
#pragma unroll
        for (int j = 0; j < 2; j++) if (len_s[lane + 32 * j] > 0) r0 = min(r0, cur0[lane + 32 * j]);
        r0 = __reduce_min_sync(0xffffffffu, r0);
        bool bad = r0 != RC_INF && r0 <= rtop - RB_WR;
        if (tid < 64 && r0 != RC_INF && !bad) {
            const int sp = my_len > 0 ? my_cmin : my_ctot;     // (also: where the chunk's events of this chain begin)
            const int lo = Wls[r0 & (RB_WR - 1)][tid];
            my_wlo = lo >= 0 ? min(lo, sp) : sp;
            if (sp - my_wlo > RC_REACH) bad = true;
            my_wld = my_wrd = min(min(my_ctot, my_wlo + RC_WN), sp + RC_LW + RC_PF);
            s_old[tid] = my_wlo; wldp[tid] = my_wld;
        }
        if (__syncthreads_or(bad)) handed = 1;
        if (!handed && r0 != RC_INF) {
            for (int cl = 0; cl < RC_CPC; cl++) {
                const int c = bx * RC_CPC + cl;
                const int before = len_s[c] > 0 ? cmin_s[c] : ctot_s[c];
                for (int sq = s_old[c] + warp; sq < wldp[c]; sq += RC_THREADS / 32) {
                    int v0, v1;
                    if (sq >= before) {
                        const int32_t *src = Q.rsg + (size_t)(coff_s[c] + sq - cmin_s[c]) * 64;
                        v0 = __ldcg(src + lane); v1 = __ldcg(src + lane + 32);
                        if (lane == 0) cevw[cl][sq & (RC_WN - 1)] = P.cev[off[c] + sq - cmin_s[c]];
                    } else {
                        const int h = __ldcg(P.gchain + c * RB_RING + (sq & (RB_RING - 1)));
                        const int a0 = lane < M ? __ldcg(P.row + (size_t)h * M + lane) : -1;
                        const int a1 = lane + 32 < M ? __ldcg(P.row + (size_t)h * M + lane + 32) : -1;
                        v0 = a0 < 0 ? -1 : P.seq[a0]; v1 = a1 < 0 ? -1 : P.seq[a1];
                    }
                    rsw[cl][sq & (RC_WN - 1)][lane] = v0; rsw[cl][sq & (RC_WN - 1)][lane + 32] = v1;
                }
            }
        }
        __syncthreads();
    }
    rc_cluster_sync();                                          // every CTA of the cluster runs before any remote store

    // ---- from here on the state of chain c lives in the registers of ONE warp: lane l of warp 0 holds chains l and l+32
    int cpos[2] = {0, 0}, ccur[2] = {RC_INF, RC_INF}, clen[2] = {0, 0}, ccmin[2] = {0, 0}, cctot[2] = {0, 0};
    int cwlo[2] = {0, 0}, cwld[2] = {0, 0}, cwrd[2] = {0, 0};
    bool ctested[2] = {false, false};
    if (warp == 0) {
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int c = lane + 32 * j;
            clen[j] = len_s[c]; ccmin[j] = cmin_s[c]; cctot[j] = ctot_s[c]; ccur[j] = cur0[c];
            if (!handed) { cwlo[j] = s_old[c]; cwld[j] = cwrd[j] = wldp[c]; }
        }
    }

    long long c_t[6] = {0, 0, 0, 0, 0, 0}, c_steps = 0, c_tests = 0, c_unk = 0;
    int stall = 0, rmin = 0;
    bool have_res = false, rows_out = false;                    // rows_out: the bulk copies of this step are issued
    // the step log (LOG only: a kernel of its own, so the marks cost the timed kernel nothing): where this launch's
    // records begin (every CTA reads it before the first exchange; CTA 0 advances it after its loop), and thread 0's
    // clock at each mark of a step
    const bool lg = LOG && tid == 0;
    if (lg) { tsm[16] = __ldcg(Q.slog); tsm[17] = __ldcg(Q.slog + 1); }
    auto mark = [&](int k) { if constexpr (LOG) { if (tid == 0) tsm[k] = (unsigned)clock64(); } };
    unsigned it = 0;                                            // steps so far (mbarrier phases)
    for (; !handed; ++it) {
        const long long t0 = clock64();
        mark(0);
        u64 (*maskbuf)[RC_MRS] = maskbuf0 + (it & 1) * 64;
        // ---- the results of the last step (every CTA holds all of them): positions, rounds, the mirror of Wf; then
        //      this step's ranges and windows.  One warp, no block-wide barrier inside.
        bool late = false;
        if (have_res) late = !rc_mbar_wait(mbar0 + 16, (it - 1) & 1);
        mark(1);
        if (tid == 0) rc_mbar_expect(mbar0 + 16, 64 * 4);      // this step's results: one word per chain
        if (rows_out) late |= !rc_mbar_wait(mbar0 + 24, (it - 1) & 1);   // the rows issued a step ago ...
        rows_out = false;
        asm volatile("cp.async.wait_all;" ::: "memory");        // ... and their event indices
        if (warp == 0) {
            bool hit[2] = {false, false}, prog = false;
            int hitseq[2] = {-1, -1};
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int c = lane + 32 * j;
                int nf = 0, base = 0;
                if (have_res && ctested[j]) {
                    const int x = xres[c], f = x >> 2, vf = x & 3;
                    base = ccmin[j] + cpos[j]; nf = f;
                    if (vf == 1) { hit[j] = true; ccur[j] = rmin + 1; hitseq[j] = base + f; }
                    cpos[j] += f;
                    prog |= f > 0 || vf == 1;
                }
                s_nfin[c] = nf; s_base[c] = base;
            }
            const int rnext = __reduce_min_sync(0xffffffffu, min(cpos[0] < clen[0] ? ccur[0] : RC_INF, cpos[1] < clen[1] ? ccur[1] : RC_INF));
            const bool anyhit = __any_sync(0xffffffffu, hit[0] || hit[1]), anyprog = __any_sync(0xffffffffu, prog);
            bool newrow = false;
            if (have_res && anyhit && rmin + 1 > rtop) {        // the hits open the mirror row of round rmin+1
                rtop = rmin + 1; newrow = true;
                if (rtop >= P.Rcap && lane == 0 && lead) atomicMin(&P.scal[SC_ERR], -5);
            }
#pragma unroll
            for (int j = 0; j < 2; j++) {                       // (each lane its own columns)
                const int c = lane + 32 * j;
                if (hit[j] && rmin + 1 < P.Rcap) {
                    Wls[(rmin + 1) & (RB_WR - 1)][c] = hitseq[j];
                    if (c / RC_CPC == bx) P.Wf[(size_t)(rmin + 1) * M + c] = cevw[c % RC_CPC][hitseq[j] & (RC_WN - 1)];
                } else if (newrow) Wls[rtop & (RB_WR - 1)][c] = -1;
            }
            int status = 0;                                     // 1: every chain is done, 2: the rest goes to k_rounds_batch
            if (rnext == RC_INF) status = 1;
            else if (rnext <= rtop - RB_WR) status = 2;
            else {
                bool moved = false;
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int c = lane + 32 * j, sp = clen[j] > 0 ? ccmin[j] + cpos[j] : cctot[j];
                    moved |= cwrd[j] != cwld[j];
                    cwrd[j] = cwld[j];
                    const int lo = Wls[rnext & (RB_WR - 1)][c];
                    cwlo[j] = max(cwlo[j], lo >= 0 ? min(lo, sp) : sp);
                    const int hi = min(min(cctot[j], cwlo[j] + RC_WN), sp + RC_LW + RC_PF), old = cwld[j];
                    if (hi > cwld[j]) { cwld[j] = hi; moved = true; }
                    const bool open = cpos[j] < clen[j];
                    const int me = lo >= 0 ? min(min(cwrd[j], open ? sp + RC_LW : cctot[j]), lo + RC_MR) : -1;
                    ctested[j] = open && ccur[j] == rnext;
                    slo[c] = lo; smend[c] = me; spos[c] = sp; s_old[c] = old; wldp[c] = cwld[j];
                    swin[c] = ctested[j] ? max(0, min(min(RC_LW, clen[j] - cpos[j]), cwrd[j] - sp)) : -1;
                    cnts[c] = lo >= 0 ? max(0, me - lo) : 0;
                    wp[c] = lo >= 0 ? lo : RC_BIG;
                }
                const bool anymoved = __any_sync(0xffffffffu, moved);
                if (have_res) stall = (anyprog || anymoved) ? 0 : stall + 1;
                if (stall >= RC_STALL) status = 2;
                else {                                          // the bytes the other CTAs will store into my mask table
                    int by = 0;
#pragma unroll
                    for (int j = 0; j < 2; j++) { const int m = lane + 32 * j; if (m / RC_CPC != bx) by += ((cnts[m] + 1) >> 1) * 16; }
                    by = __reduce_add_sync(0xffffffffu, by);
                    if (lane == 0) rc_mbar_expect(mbar0 + 8 * (it & 1), (unsigned)by);
                }
            }
            if (lane == 0) { ws[0] = rnext; ws[1] = status; }
        }
        mark(2);
        const bool timed_out = __syncthreads_or(late);          // (never, unless a peer CTA died)
        const int rprev = rmin, status = ws[1];
        rmin = ws[0];
        if (timed_out || status != 0) {
            if (have_res && !timed_out && tid < RC_CPC * RC_LW) {   // final rounds of the last step
                const int cl = tid / RC_LW, j = tid % RC_LW, c = bx * RC_CPC + cl;
                if (j < s_nfin[c]) P.round[cevw[cl][(s_base[c] + j) & (RC_WN - 1)]] = rprev;
            }
            if (timed_out && tid == 0 && lead) atomicMin(&P.scal[SC_ERR], -4);
            if (timed_out || status == 2) handed = 1;
            break;
        }
        const long long t1 = clock64();
        mark(3);
        // ---- a: the masks of my members' ranges into my own table (4 warps per member), then each member's masks to
        //         every other CTA as one wide store per (member, CTA).  Bit b of a mask's low word is column 2b, of its
        //         high word column 2b+1: the tests only COUNT columns.
        {
            const int cl = warp / RC_WPC, c = bx * RC_CPC + cl, lo = slo[c], cnt = cnts[c];
            const int2 wv = reinterpret_cast<const int2 *>(wp)[lane];
            for (int i0 = warp % RC_WPC; i0 < cnt; i0 += 4 * RC_WPC) {      // four rows in flight
                int2 v[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int i = i0 + u * RC_WPC;
                    v[u] = i < cnt ? reinterpret_cast<const int2 *>(rsw[cl][(lo + i) & (RC_WN - 1)])[lane] : make_int2(-1, -1);
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int i = i0 + u * RC_WPC;
                    if (i < cnt) {                              // (warp-uniform)
                        const unsigned b0 = __ballot_sync(0xffffffffu, v[u].x >= wv.x), b1 = __ballot_sync(0xffffffffu, v[u].y >= wv.y);
                        if (lane == 0) maskbuf[c][i] = (u64)b0 | (u64)b1 << 32;
                    }
                }
            }
            mark(4);
            if (tid < RC_CPC * 64) {                            // {threshold (+1 on the chain's own column: its self-parent), span}
                const int cl2 = tid >> 6, m = tid & 63;
                cst[cl2][m] = make_int2(wp[m] + (m == bx * RC_CPC + cl2 ? 1 : 0), cnts[m]);
            }
            __syncthreads();
            mark(5);
            for (int pair = warp; pair < RC_CPC * RC_CS; pair += RC_THREADS / 32) {
                const int cl2 = pair & (RC_CPC - 1), r = pair / RC_CPC, c2 = bx * RC_CPC + cl2;
                if (r == bx || 2 * lane >= cnts[c2]) continue;
                const uint4 val = *reinterpret_cast<const uint4 *>(&maskbuf[c2][2 * lane]);
                rc_sta_v4(rc_map(&maskbuf[c2][2 * lane], (unsigned)r), val, rc_map(iv + 2304 + 2 * (it & 1), (unsigned)r));
            }
        }
        const long long t2 = clock64();
        mark(6);
        // off the path the other CTAs wait on: the final rounds of the last step, the next rows of my chains' windows
        mark(13);
        if (have_res && tid < RC_CPC * RC_LW) {
            const int cl = tid / RC_LW, j = tid % RC_LW, c = bx * RC_CPC + cl;
            if (j < s_nfin[c]) P.round[cevw[cl][(s_base[c] + j) & (RC_WN - 1)]] = rprev;
        }
        // the rows of chain cl by lane 0 of warp 5 cl (one warp per SM sub-partition), as one or two bulk copies (the
        // window is a ring) that count their bytes on the rows' mbarrier; its event indices by the same warp.  Rows that
        // a later row of the same step overwrites in the ring are never read: only the last RC_WN are copied.
        if (warp % 5 == 0 && warp < 5 * RC_CPC) {
            const int cl = warp / 5, c = bx * RC_CPC + cl, n = wldp[c] - s_old[c];
            const int nrow = max(0, min(n, RC_WN)), lo2 = s_old[c] + max(0, n - RC_WN);
            const size_t g = (size_t)(coff_s[c] + lo2 - cmin_s[c]);
            if (lane == 0) {
                rc_mbar_expect(mbar0 + 24, (unsigned)nrow * 256u);
                if (nrow > 0) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // (after the generic reads of the slots)
                    const int s0 = lo2 & (RC_WN - 1), n0 = min(nrow, RC_WN - s0);
                    rc_bulk(rsw[cl][s0], Q.rsg + g * 64, (unsigned)n0 * 256u, mbar0 + 24);
                    if (nrow > n0) rc_bulk(rsw[cl][0], Q.rsg + (g + n0) * 64, (unsigned)(nrow - n0) * 256u, mbar0 + 24);
                }
            }
            for (int i = lane; i < nrow; i += 32) rc_cp4(&cevw[cl][(lo2 + i) & (RC_WN - 1)], P.cev + off[c] + (lo2 - cmin_s[c]) + i);
        }
        rows_out = true;
        asm volatile("cp.async.commit_group;" ::: "memory");
        mark(14);
        long long t3;
        // ---- b: first pending event with P_r (1) or beyond the masks (2), per chain
        if (UNIT) {
            // every position of the window at once, bit-sliced: 8 tests per warp, 4 lanes x 16 members per test.  A lane
            // adds the masks of its live members into a vertical counter (one bit plane per power of two, 64 columns
            // wide), the 4 lanes of a test add their counters, and the column counts are compared with the threshold
            // plane by plane -- no transposes.  What needs only MY rows runs before the wait for the others' masks.
            const int cl = warp / RC_WPC, c = bx * RC_CPC + cl;
            const int q = lane >> 2, pp = lane & 3, t = (warp % RC_WPC) * 8 + q;
            const bool act = t < swin[c];
            const int thr_i = (int)thr;
            const int sq = spos[c] + t;
            const char *rowb = reinterpret_cast<const char *>(rsw[cl][sq & (RC_WN - 1)]) + 64 * pp;
            const char *cstb = reinterpret_cast<const char *>(cst[cl]) + 128 * pp;
            const int r4 = (2 * q + (pp >> 1)) * 4;            // (the 32 lanes start at 32 different banks)
            int offs[16], neg = 0;
            bool unk = false;
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const int bo = (4 * i + r4) & 60;               // member 16 pp + bo / 4
                const int pr = *reinterpret_cast<const int *>(rowb + bo);
                const int2 cs = *reinterpret_cast<const int2 *>(cstb + 2 * bo);
                const int o2 = act ? pr - cs.x : -1;            // >= 0: the member is live, its mask is maskbuf[m][o2]
                unk |= o2 >= cs.y;                             // ... unless the event lies beyond the prepared masks
                neg += o2 >> 31;
                offs[i] = max(o2, -1);
            }
            int lv = 16 + neg;
            lv += __shfl_xor_sync(0xffffffffu, lv, 1);
            lv += __shfl_xor_sync(0xffffffffu, lv, 2);
            const unsigned ub = __ballot_sync(0xffffffffu, unk);
            unk = ((ub >> (lane & ~3)) & 0xfu) != 0;
            const bool need = act && lv > thr_i && !unk;       // (lv <= thr: hits[c_] <= the live members)
            int v = (act && lv > thr_i && unk) ? 2 : 0;
            mark(7);
            late = !rc_mbar_wait(mbar0 + 8 * (it & 1), (it >> 1) & 1);
            t3 = clock64();
            mark(8);
            if (__any_sync(0xffffffffu, need)) {
                c_tests++;
                u64 x[16];
#pragma unroll
                for (int i = 0; i < 16; i++) {
                    const int m = 16 * pp + (((4 * i + r4) & 60) >> 2);
                    x[i] = (need && offs[i] >= 0) ? maskbuf[m][offs[i]] : 0ull;
                }
                u64 a[8], t2a, t2b, t4a, t4b, t8a, t8b;
                a[0] = a[1] = a[2] = a[3] = 0;
                rc_csa(t2a, a[0], a[0], x[0], x[1]);   rc_csa(t2b, a[0], a[0], x[2], x[3]);   rc_csa(t4a, a[1], a[1], t2a, t2b);
                rc_csa(t2a, a[0], a[0], x[4], x[5]);   rc_csa(t2b, a[0], a[0], x[6], x[7]);   rc_csa(t4b, a[1], a[1], t2a, t2b);
                rc_csa(t8a, a[2], a[2], t4a, t4b);
                rc_csa(t2a, a[0], a[0], x[8], x[9]);   rc_csa(t2b, a[0], a[0], x[10], x[11]); rc_csa(t4a, a[1], a[1], t2a, t2b);
                rc_csa(t2a, a[0], a[0], x[12], x[13]); rc_csa(t2b, a[0], a[0], x[14], x[15]); rc_csa(t4b, a[1], a[1], t2a, t2b);
                rc_csa(t8b, a[2], a[2], t4a, t4b);
                rc_csa(a[4], a[3], a[3], t8a, t8b);           // 16 a[4] + 8 a[3] + 4 a[2] + 2 a[1] + a[0] = members per column
                rc_vadd_xor<5>(a, 1);
                rc_vadd_xor<6>(a, 2);                          // 7 planes: 0..64 per column
                u64 gt = 0, eq = ~0ull;
#pragma unroll
                for (int k = 6; k >= 0; k--) {
                    const u64 tk = ((thr_i >> k) & 1) ? ~0ull : 0ull;
                    gt |= eq & a[k] & ~tk;
                    eq &= ~(a[k] ^ tk);
                }
                if (need) v = __popcll(gt) > thr_i ? 1 : 0;    // a COUNT of members against the STAKE threshold (quirk Q3)
            }
            if (v == 2) c_unk++;
            if (pp == 0) vres[cl * RC_LW + t] = v;
            const int w2 = warp < RC_CPC ? swin[bx * RC_CPC + warp] : -1;   // (read before the barrier: warp 0 rewrites swin right after it)
            mark(9);
            if (__syncthreads_or(late)) {
                if (tid == 0 && lead) atomicMin(&P.scal[SC_ERR], -4);
                handed = 1;
                break;
            }
            mark(10);
            if (warp < RC_CPC) {
                const int c2 = bx * RC_CPC + warp;
                const int x = vres[warp * RC_LW + lane];
                const unsigned inwin = w2 >= 32 ? 0xffffffffu : (w2 > 0 ? (1u << w2) - 1u : 0u);
                const unsigned nz = __ballot_sync(0xffffffffu, x != 0) & inwin;
                const int f = nz ? __ffs(nz) - 1 : max(w2, 0);
                const int vf = nz ? __shfl_sync(0xffffffffu, x, f & 31) : 0;
                if (lane < RC_CS) {
                    const unsigned xv = w2 >= 0 ? (unsigned)(f << 2 | vf) : 0u;
                    rc_sta_u32(rc_map(&xres[c2], (unsigned)lane), xv, rc_map(iv + 2304 + 4, (unsigned)lane));
                }
            }
        } else {
            mark(7);
            late = !rc_mbar_wait(mbar0 + 8 * (it & 1), (it >> 1) & 1);
            mark(8); mark(9);
            if (__syncthreads_or(late)) {
                if (tid == 0 && lead) atomicMin(&P.scal[SC_ERR], -4);
                handed = 1;
                break;
            }
            t3 = clock64();
            mark(10);
            // integer stakes: a 5-ary search with the chain's 4 warps, one test of swirld_rounds.cuh's kind per warp and pass
            if (tid < RC_CPC) { sa[tid] = -1; sb[tid] = max(swin[bx * RC_CPC + tid], 0); svb[tid] = 0; }
            __syncthreads();
            for (int pass = 0; pass < RC_PASSES; pass++) {
                const int cl = warp / RC_WPC, i = warp % RC_WPC, c = bx * RC_CPC + cl;
                const int a = sa[cl], b = sb[cl], nun = b - a - 1;
                int t = -1;
                if (swin[c] > 0 && nun > 0) {
                    if (nun < RC_WPC) { if (i < nun) t = a + 1 + i; }
                    else t = a + ((i + 1) * (nun + 1)) / (RC_WPC + 1);
                }
                int v = 0;
                if (t >= 0) {                                   // (warp-uniform)
                    c_tests++;
                    const int sq = spos[c] + t;
                    const int *row = rsw[cl][sq & (RC_WN - 1)];
                    int pre[2], W[2];
                    bool live[2];
                    i64 lv = 0;
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        const int m = lane + 32 * j;
                        pre[j] = m == c ? sq - 1 : row[m];      // the own column is set back to the self-parent
                        W[j] = slo[m];
                        live[j] = W[j] >= 0 && pre[j] >= W[j];
                        i64 sv = live[j] ? stake_s[m] : 0;
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) sv += __shfl_xor_sync(0xffffffffu, sv, o);
                        lv += sv;
                    }
                    if (lv > thr) {                             // else: hits[c_] <= stake of the live members
                        const bool unk = (live[0] && pre[0] >= smend[lane]) || (live[1] && pre[1] >= smend[lane + 32]);
                        if (__any_sync(0xffffffffu, unk)) { v = 2; c_unk++; }
                        else {
                            u64 mm[2];
#pragma unroll
                            for (int j = 0; j < 2; j++) mm[j] = live[j] ? maskbuf[lane + 32 * j][pre[j] - W[j]] : 0ull;
                            unsigned T[2][2];                   // T[jj][j]: bit b = member jj*32+b sees the column of bit (j, lane)
#pragma unroll
                            for (int jj = 0; jj < 2; jj++)
#pragma unroll
                                for (int j = 0; j < 2; j++) T[jj][j] = rb_transpose32((unsigned)(mm[jj] >> (32 * j)), lane);
                            int cntc = 0;
#pragma unroll
                            for (int j = 0; j < 2; j++) {
                                i64 hits = 0;
#pragma unroll
                                for (int jj = 0; jj < 2; jj++)
#pragma unroll 8
                                    for (int bq = 0; bq < 32; bq++) hits += ((T[jj][j] >> bq) & 1) ? stake_s[jj * 32 + bq] : 0;
                                cntc += __popc(__ballot_sync(0xffffffffu, hits > thr));
                            }
                            v = (i64)cntc > thr ? 1 : 0;       // a COUNT of members against the STAKE threshold (quirk Q3)
                        }
                    }
                }
                if (lane == 0) tres[cl * RC_WPC + i] = t >= 0 ? (t << 2 | v) : -1;
                __syncthreads();
                if (tid < RC_CPC) {
                    int a2 = sa[tid], b2 = sb[tid], vb2 = svb[tid];
#pragma unroll
                    for (int q = 0; q < RC_WPC; q++) {
                        const int x = tres[tid * RC_WPC + q];
                        if (x < 0) continue;
                        const int tq = x >> 2, vq = x & 3;
                        if (vq == 0) a2 = max(a2, tq);
                        else if (tq < b2) { b2 = tq; vb2 = vq; }
                    }
                    sa[tid] = a2; sb[tid] = b2; svb[tid] = vb2;
                }
                __syncthreads();
            }
            if (tid < RC_CPC * RC_CS) {                         // (first position, what it is) of my chains to every CTA
                const int cl = tid & (RC_CPC - 1), rank = tid / RC_CPC, c = bx * RC_CPC + cl;
                unsigned x = 0;
                if (swin[c] >= 0) { const int f = sb[cl]; x = (unsigned)(f << 2 | (f < swin[c] ? svb[cl] : 0)); }
                rc_sta_u32(rc_map(&xres[c], (unsigned)rank), x, rc_map(iv + 2304 + 4, (unsigned)rank));
            }
        }
        const long long t4 = clock64();
        mark(11);
        const long long t5 = clock64();
        have_res = true;
        c_t[0] += t1 - t0; c_t[1] += t2 - t1; c_t[2] += t3 - t2; c_t[3] += t4 - t3; c_t[4] += t5 - t4;
        c_steps++;
        if constexpr (LOG) if (lg && tsm[16] + it < tsm[17]) {
            unsigned *o = Q.slog + RC_LOGH + ((size_t)(tsm[16] + it) * RC_CS + bx) * RC_NLOG;
            const unsigned dfr = tsm[14] - tsm[13];
            o[RL_WAIT] = tsm[1] - tsm[0]; o[RL_CTL] = tsm[2] - tsm[1]; o[RL_BAR1] = tsm[3] - tsm[2];
            o[RL_MASK] = tsm[4] - tsm[3]; o[RL_BAR2] = tsm[5] - tsm[4]; o[RL_PUSH] = tsm[6] - tsm[5];
            o[RL_TEST1] = tsm[7] - tsm[6] - dfr; o[RL_MWAIT] = tsm[8] - tsm[7]; o[RL_TEST2] = tsm[9] - tsm[8];
            o[RL_BAR3] = tsm[10] - tsm[9]; o[RL_SEND] = tsm[11] - tsm[10]; o[RL_DEFER] = dfr;
            o[RL_SENDER] = tsm[6] - tsm[1]; o[RL_TESTER] = tsm[11] - tsm[8];
        }
    }
    if (rows_out) (void)rc_mbar_wait(mbar0 + 24, it & 1);    // (the loop was left inside the tests)
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    if (lead) {
        if (warp == 0) {
#pragma unroll
            for (int j = 0; j < 2; j++) { Q.cont[lane + 32 * j] = cpos[j]; Q.cont[64 + lane + 32 * j] = ccur[j]; }
        }
        if (tid == 0) {
            Q.cont[128] = handed;
            if (P.n > 0) P.scal[SC_MAX_ROUND] = rtop;
        }
    }
    if (P.dbg && lane == 0) {
        atomicAdd((unsigned long long *)P.dbg + 11, (unsigned long long)c_tests);     // (the slots of k_rounds_batch's counters)
        atomicAdd((unsigned long long *)P.dbg + 12, (unsigned long long)c_unk);
    }
    if (P.dbg && tid == 0 && lead) {
        unsigned long long *o = (unsigned long long *)P.dbg;
        for (int i = 0; i < 6; i++) atomicAdd(&o[i], (unsigned long long)c_t[i]);
        atomicAdd(&o[6], (unsigned long long)c_steps);
        atomicAdd(&o[7], 1ull);                                 // launches, and how many handed work back
        atomicAdd(&o[15], (unsigned long long)handed);
    }
    if constexpr (LOG) if (lg && lead) Q.slog[0] = tsm[16] + (unsigned)c_steps;     // (the next launch's records follow this one's)
    rc_cluster_sync();                                          // nobody leaves while its shared memory may still be written
}

// several independent node-views (swirld_rounds.cuh, k_rounds_batch): one cluster per view (blockIdx.y), as many side
// by side as the device holds -- the clusters never talk to each other, so this is an ordinary (non-cooperative) launch
template <bool UNIT, class Src>
__global__ void __launch_bounds__(RC_THREADS, 1) k_rounds_cluster(Src s) { rounds_cluster_body<UNIT, false>(params(s)); }
// the same with the per-CTA step log (RcParams::slog), for one view: launched instead of k_rounds_cluster<UNIT, RcParams>
// when the engine keeps the log
template <bool UNIT>
__global__ void __launch_bounds__(RC_THREADS, 1) k_rounds_cluster_log(RcParams q) { rounds_cluster_body<UNIT, true>(q); }
SW_SRC_INSTANCES_OF(k_rounds_cluster, RcParams, false) SW_SRC_INSTANCES_OF(k_rounds_cluster, RcParams, true)
