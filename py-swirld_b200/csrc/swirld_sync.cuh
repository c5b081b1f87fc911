// swirld_sync.cuh -- the sending end of Node.sync on the GPU: the requester's summary and the responder's reply.
//
// In a responder view with head H, row(H)[c] is the latest event of member c that H sees (-1: none), and S[c] the
// requester's summary: the height of the latest c-event its head sees, -1 if none (swirld.py:125-126).  ask_sync's
// BFS from H over the parents the requester lacks (swirld.py:154-161, utils.py:24-34) selects
//
//     reply(H, S) = {H} u { x < H : x <= row(H)[creator x]  and  (S[creator x] = -1  or  height[x] > S[creator x]) }
//
// On a fork-free graph the ancestors of H by member c are c's chain up to row(H)[c]; "the requester does not see x" is
// closed towards descendants, so every path from H to such an x runs through such events only and the BFS reaches
// it; and bfs yields its start whatever the filter says.  The equality needs S from a view of the same fork-free
// gossip (what the protocol sends): for an arbitrary S the closed form may select events the BFS cannot reach.
//
// The reply is a stream compaction over [0, H] of each view, count then scatter, in three launches however many views
// and events: k_sync_count counts each tile's selected events, k_sync_scan (one CTA) turns the counts of every view's
// tiles into output positions, and k_sync_select selects again and writes each selected event's columns at its
// position, in ascending index order (a topological order of the responder: sw_ingest takes it as it is).  Each pass
// reads creator and height once, 8 bytes per event, plus the selected rows.  The kernels take their parameters from a
// Src (swirld_kernels.cuh, params): one view by value, or the device array of the views with blockIdx.y the view.
#pragma once
#include "swirld_kernels.cuh"

constexpr int SY_THREADS = 256;
constexpr int SY_TILE = 2048;        // events per CTA of k_sync_count / k_sync_select

struct SyncParams {
    const int32_t *row, *height, *creator, *p0, *p1;   // the view's columns (row: its can_see table, M per event)
    const double *t;
    const uint8_t *sig;
    const int32_t *summary;          // the requester's S: M entries
    int32_t *heights_out;            // k_sync_summary: M entries
    int32_t *tile_cnt;               // the call's tile counts, every view's tiles in view order
    const int32_t *tile_off;         // ... their exclusive prefix (k_sync_scan)
    const int32_t *fits;             // k_sync_scan: 1 when the whole reply fits the caller's capacity
    int32_t *o_index, *o_creator, *o_p0, *o_p1;        // the packed output block: every view's rows, in view order
    double *o_t;
    uint8_t *o_sig;
    int M, head, tile0, ntiles;      // tile0: the view's first tile among the call's
};

// the requester's summary for head H: height[row(H)[c]] for every member c, -1 where H sees none of c's events
template <class Src>
__global__ void __launch_bounds__(SY_THREADS) k_sync_summary(Src s) {
    const SyncParams &P = params(s);
    const int32_t *r = P.row + (size_t)P.head * P.M;
    for (int c = threadIdx.x; c < P.M; c += blockDim.x) {
        const int x = r[c];
        P.heights_out[c] = x < 0 ? -1 : P.height[x];
    }
}

// row(H) and S staged in shared memory (2 x 4 KB at M = 1024)
__device__ __forceinline__ void sync_stage(const SyncParams &P, int *rs, int *ss) {
    const int32_t *r = P.row + (size_t)P.head * P.M;
    for (int c = threadIdx.x; c < P.M; c += blockDim.x) { rs[c] = r[c]; ss[c] = P.summary[c]; }
    __syncthreads();
}

__device__ __forceinline__ bool sync_pick(const SyncParams &P, const int *rs, const int *ss, int x) {
    if (x > P.head) return false;
    if (x == P.head) return true;
    const int c = P.creator[x], s = ss[c];
    return x <= rs[c] && (s < 0 || P.height[x] > s);
}

template <class Src>
__global__ void __launch_bounds__(SY_THREADS) k_sync_count(Src s) {
    const SyncParams &P = params(s);
    if ((int)blockIdx.x >= P.ntiles) return;
    extern __shared__ int sy_smem[];
    int *rs = sy_smem, *ss = sy_smem + P.M;
    sync_stage(P, rs, ss);
    const int base = blockIdx.x * SY_TILE;
    int cnt = 0;
    for (int k = 0; k < SY_TILE; k += SY_THREADS)
        cnt += __syncthreads_count(sync_pick(P, rs, ss, base + k + threadIdx.x));
    if (threadIdx.x == 0) P.tile_cnt[P.tile0 + blockIdx.x] = cnt;
}

// One CTA: the exclusive prefix of the T tile counts (tile_off, T + 1 entries); the header of the output block,
// [total, count of view 0 .. B-1, offset of view 0 .. B]; fits = total <= cap.  tile0: B + 1 entries.
__global__ void __launch_bounds__(1024) k_sync_scan(const int32_t *tile_cnt, int T, const int32_t *tile0, int B, int cap,
                                                    int32_t *tile_off, int32_t *fits, int32_t *hdr) {
    __shared__ int wsum_s[32];
    __shared__ int carry;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < T; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const int v = i < T ? tile_cnt[i] : 0;
        int x = v;
        for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
        if (lane == 31) wsum_s[w] = x;
        __syncthreads();
        if (w == 0) {
            int y = lane < nw ? wsum_s[lane] : 0;
            for (int d = 1; d < 32; d <<= 1) { const int z = __shfl_up_sync(0xffffffffu, y, d); if (lane >= d) y += z; }
            if (lane < nw) wsum_s[lane] = y;
        }
        __syncthreads();
        const int c0 = carry;
        if (i < T) tile_off[i] = c0 + x - v + (w ? wsum_s[w - 1] : 0);
        __syncthreads();
        if (threadIdx.x == 0) carry = c0 + wsum_s[nw - 1];
        __syncthreads();
    }
    const int total = carry;
    if (threadIdx.x == 0) { tile_off[T] = total; hdr[0] = total; *fits = total <= cap; }
    __syncthreads();
    for (int v = threadIdx.x; v < B; v += blockDim.x) {
        const int a = tile_off[tile0[v]], b = tile_off[tile0[v + 1]];
        hdr[1 + v] = b - a;
        hdr[1 + B + v] = a;
    }
    if (threadIdx.x == 0) hdr[1 + 2 * B] = total;
}

// Select again, and write each selected event's index, creator, parents, t and signature at its position
template <class Src>
__global__ void __launch_bounds__(SY_THREADS) k_sync_select(Src s) {
    const SyncParams &P = params(s);
    if ((int)blockIdx.x >= P.ntiles || !*P.fits) return;
    extern __shared__ int sy_smem[];
    int *rs = sy_smem, *ss = sy_smem + P.M;
    __shared__ int wcnt[SY_THREADS / 32];
    sync_stage(P, rs, ss);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int base = blockIdx.x * SY_TILE;
    int at = P.tile_off[P.tile0 + blockIdx.x];
    for (int k = 0; k < SY_TILE; k += SY_THREADS) {
        const int x = base + k + threadIdx.x;
        const bool pick = sync_pick(P, rs, ss, x);
        const unsigned m = __ballot_sync(0xffffffffu, pick);
        if (lane == 0) wcnt[w] = __popc(m);
        __syncthreads();
        int before = 0, all = 0;
        for (int j = 0; j < SY_THREADS / 32; j++) { before += j < w ? wcnt[j] : 0; all += wcnt[j]; }
        if (pick) {
            const int o = at + before + __popc(m & ((1u << lane) - 1));
            P.o_index[o] = x; P.o_creator[o] = P.creator[x]; P.o_p0[o] = P.p0[x]; P.o_p1[o] = P.p1[x]; P.o_t[o] = P.t[x];
            const uint4 *src = reinterpret_cast<const uint4 *>(P.sig + (size_t)64 * x);
            uint4 *dst = reinterpret_cast<uint4 *>(P.o_sig + (size_t)64 * o);
#pragma unroll
            for (int q = 0; q < 4; q++) dst[q] = src[q];
        }
        at += all;
        __syncthreads();
    }
}
