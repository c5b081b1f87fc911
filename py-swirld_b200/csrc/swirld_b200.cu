// swirld_b200.cu -- host side of libswirld_b200.so: the C ABI of include/swirld_b200.h
// over the kernels in swirld_*.cuh.  No torch, no CPU compute path: every
// consensus result is produced by a kernel; the host only validates the graph shape
// on append (what Node.is_valid_event checks, swirld.py:104-108), keeps the
// creator/height/chain-position mirrors it needs for that, and moves bytes.
#include "swirld_kernels.cuh"
#include "swirld_cansee.cuh"
#include "swirld_rounds.cuh"
#include "swirld_rcluster.cuh"
#include "swirld_wide.cuh"
#include "swirld_stream.cuh"
#include "swirld_verify.cuh"
#include "swirld_sign.cuh"
#include "swirld_sync.cuh"

#include <cstdlib>
#include "../../include/swirld_b200.h"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <array>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

namespace {

std::string g_create_error;

// 32-byte event ids (BLAKE2b, swirld.py:95) -> arrival index
using Id32 = std::array<uint64_t, 4>;
struct Id32Hash { size_t operator()(const Id32 &k) const { return (size_t)(k[0] ^ (k[1] * 0x9E3779B97F4A7C15ull)); } };

// ---- the owners of the engine's CUDA resources: move-only, released on destruction
// Device memory, or pinned host memory (PINNED): cap() elements of T, at least one (a zero-size request gets one)
template <class T, bool PINNED = false>
class Mem {
    T *p_ = nullptr;
    size_t n_ = 0;
  public:
    Mem() = default;
    Mem(Mem &&o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    Mem &operator=(Mem &&o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
    ~Mem() { reset(); }
    T *get() const { return p_; }
    size_t cap() const { return n_; }
    void reset() {
        if (p_) (void)(PINNED ? cudaFreeHost(p_) : cudaFree(p_));
        p_ = nullptr; n_ = 0;
    }
    cudaError_t alloc(size_t n) {
        reset();
        void *q = nullptr;
        const size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
        const cudaError_t s = PINNED ? cudaMallocHost(&q, bytes) : cudaMalloc(&q, bytes);
        if (s == cudaSuccess) { p_ = static_cast<T *>(q); n_ = std::max<size_t>(n, 1); }
        return s;
    }
};
template <class T> using Pinned = Mem<T, true>;

// A stream, an event or a peer's IPC-mapped memory
template <class H, cudaError_t (*Release)(H)>
class Handle {
    H h_ = nullptr;
  protected:
    // `h` by reference: it is read only once the call that made `s` has written it
    cudaError_t take(cudaError_t s, const H &h) { reset(); if (s == cudaSuccess) h_ = h; return s; }
  public:
    Handle() = default;
    Handle(Handle &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Handle &operator=(Handle &&o) noexcept { std::swap(h_, o.h_); return *this; }
    ~Handle() { reset(); }
    H get() const { return h_; }
    void reset() { if (h_) (void)Release(h_); h_ = nullptr; }
};
struct Stream : Handle<cudaStream_t, cudaStreamDestroy> {
    cudaError_t create() { cudaStream_t s = nullptr; return take(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking), s); }
};
struct Event : Handle<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(bool timing = false) {
        cudaEvent_t ev = nullptr;
        return take(timing ? cudaEventCreate(&ev) : cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), ev);
    }
};
struct PeerMem : Handle<void *, cudaIpcCloseMemHandle> {
    cudaError_t open(const void *handle64) {
        cudaIpcMemHandle_t h;
        memcpy(&h, handle64, sizeof h);
        void *p = nullptr;
        return take(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), p);
    }
};

// What the time of a span counts towards (fold_spans).  `scan`: a can_see scan outside any divide span, whose time is
// divide time too; `scan_in_divide`: one inside a divide span, which counts it already; `rounds`: the round kernels.
enum class SpanCat { divide, fame, order, scan, rounds, scan_in_divide };

// `a` is `own_a`, or the start of another span, which owns it
struct TimedSpan { cudaEvent_t a; Event own_a, b; SpanCat cat; };

// The round stream (SW_ROUNDS_AHEAD, M <= 64, calls that go to the cluster kernel): a call whose can_see rows reach
// beyond its end starts the round kernels of the next piece of events on `stream`, which then runs beside the call's
// finish and fame kernels and the host's turn-around.  Round numbers are a function of the graph alone, so a piece
// writes the final rounds of its events.  Only the rs_* functions and divide_ahead write these fields.  While `synced`:
// - The pieces are contiguous and cover [n_divided, rounded).  A piece may span several calls; `pieces` holds those
//   that end beyond the last call, in order.
// - What the engine shows a caller (Wf, the ring, the counts, the round top, errors) stays the compute stream's, and
//   only the compute stream writes it.  The round stream's kernels write copies of their own: `Wf`, `gchain` (the
//   ring), `meta` (two chunk meta blocks: counts, offsets, barrier, witness count) and `scal` (round top, error slot);
//   the finish kernels of each call publish the call's part of them (RbFold).
// - Every piece ends with an event of its own.  The end of the last piece has one owner at any time: `pieces` until a
//   call has waited for the piece, then `tail`, and `free` only once a newer piece has its own end.  So rs_drain finds
//   it in one of the first two, and an event in `free` is recorded again only as the end of a newer piece.
// - A piece's k_rb_prep runs on `prep`, beside the cluster kernel of the piece before it, into the meta block and the
//   d_rsg buffer that piece does not use (`buf` alternates).  It waits for the piece before that one to have finished
//   with them (`bufdone`), and the piece's cluster kernel waits for it (`prepped`).  d_rsg[0] is the compute stream's
//   buffer too, which has it back after the wait of rs_drain.
// - The round stream's ring takes a piece's events in a launch of its own at the end of the piece (k_rb_ring): the
//   only readers of the ring slots it overwrites are this piece's cluster kernel and hand-over, which are before it on
//   the same stream, and the next piece's kernels, which are after it; the preps never read the ring.  So no reader
//   sees a slot overwritten too early or too late.
struct RoundStream {
    bool on = false;
    Stream stream, prep;          // the round stream and its prep stream
    Event wait;                   // both go on after what the compute stream had been given (rs_follow)
    Event prepped[2], bufdone[2];
    int buf = 0;                  // the buffers of the next piece
    struct Piece { int end; Event done; };
    std::vector<Piece> pieces;    // the pieces that end beyond the last call, in order
    Event tail;                   // the end of the last piece, once a call has waited for it (then `pieces` is empty)
    std::vector<Event> free;      // ends of older pieces, for newer ones to use
    Mem<int32_t> Wf, gchain, meta, scal;
    bool synced = false;          // the copies hold everything below `rounded`
    int rounded = 0;              // events rounded so far (the last piece ends here)
    unsigned epoch = 0;           // launches on the round stream (mask-cache keys of their own: the top bit set)
    int wslot = 0;                // which of the two witness counts of d_rbmeta the next call uses
};

}  // namespace

struct sw_engine {
    int M = 0, NC = 1, cap = 0, C = 6, device = 0, Rcap = 0;
    int NJ = 1;                   // words per member set on the wide path: next power of two >= ceil(M/32)
    int MS = 64;                  // per-round array stride of find_order (64, or M on the wide path)
    int MP = 64;                  // max(M, 64): size of the per-member scratch arrays
    bool wide = false;            // swirld_wide.cuh kernels (M > 64, or SW_FORCE_WIDE=1)
    bool unit = true;
    i64 tot = 0;
    std::vector<i64> h_stake;
    Stream stream;
    Stream copy_stream;                              // sw_append's copies run beside the kernels of earlier chunks
    // host mirrors for validation / views
    std::vector<int32_t> h_creator, h_head, h_count;
    Pinned<int32_t> h_height, h_seq;                 // cap entries: sources of asynchronous copies
    Pinned<uint8_t> h_stale;                         // the other-parent is not its member's latest event
    // h_count as it stood after every SNAP-th event and at the end of every append not yet divided, so that the
    // per-member counts of any chunk cost O(M) plus fewer than SNAP events (chunk_prep)
    static constexpr int SNAP = 4096;
    std::vector<int> snap_at;                        // event counts of the snapshots, ascending
    std::vector<int32_t> snap_cnt;                   // [snapshot][M]
    size_t snap_kept = 0;                            // snapshots [0, snap_kept) are all SNAP-event ones
    struct PendingAppend { int base; Event done; };
    std::vector<PendingAppend> appends;              // copies (+ eager can_see scans) the compute stream has not waited for yet
    Event scan_ev;                                   // last can_see scan issued on the compute stream
    bool scan_ev_set = false;
    int n_events = 0, n_divided = 0, n_tx = 0;
    // device columns
    Mem<int32_t> d_p0, d_p1, d_creator, d_seq, d_height;
    Mem<uint8_t> d_stale;
    Mem<long long> d_dbg;
    unsigned rb_epoch = 0;        // launches of the round kernel (mask-cache key)
    int n_sm = 0;
    Mem<int32_t> d_Wf, d_cev, d_rbmeta, d_rbtot, d_gchain;   // round-batch state (d_rbmeta: rb_meta)
    Mem<ulonglong2> d_sc;
    Mem<uint8_t> d_res;
    // cluster round kernel (swirld_rcluster.cuh): seq-space rows of the current chunk, 64 ints per event (the round
    // stream's pieces use both buffers in turn, the compute stream the first), hand-over state
    Mem<int32_t> d_rsg[2], d_rccont;
    Mem<unsigned> d_rcslog;       // the cluster kernel's per-CTA step log (SW_RC_STEPS; empty otherwise)
    bool rc_ok = false;           // a 16-CTA cluster with its shared memory can be resident on this device
    int rc_min_n = 2048;          // shorter chunks go to the grid-wide kernel directly
    RoundStream rs;
    Mem<RcParams> d_rcviews;
    Mem<RbParams> d_views;        // sw_batch_divide_rounds: the views' parameters (owned by the first engine of a batch)
    Event view_ev;
    // sw_batch_decide_fame / sw_batch_find_order (owned by the first engine of a batch): the views' parameters, rounds
    // and gathered scalars, laid out per call in one device block and its pinned host mirror
    Mem<char> d_vbuf;
    Pinned<char> h_vbuf;
    int n_rowed = 0;              // events whose can_see row is complete
    // can_see scan scratch (swirld_cansee.cuh)
    Mem<int4> d_cs_meta;
    Mem<uint8_t> d_cs_wr, d_cs_xb, d_cs_sflag;
    Mem<int32_t> d_cs_last, d_cs_Q, d_cs_carry, d_cs_slow, d_cs_slowcnt, d_cs_xlist, d_cs_slowblk, d_cs_blkcnt;
    std::vector<int32_t> h_stale_cum;    // h_stale_cum[i] = stale other-parents among events [0, i)
    int cs_min_B = 256;           // smallest block length the scan uses (sizes the per-block scratch)
    Mem<double> d_t;
    Mem<uint8_t> d_sig;
    Mem<int32_t> d_row, d_round;
    Mem<u64> d_SM;
    Mem<uint8_t> d_wit;
    Mem<int8_t> d_famous_ev;
    // wide path
    Mem<unsigned> d_scw, d_SMw, d_Sw;
    Mem<u64> d_sctag, d_hitmin;
    // several GPUs (sw_peer_connect): tests of a round step sharded by chain, first hits exchanged over NVLink
    int rank = 0, nranks = 1;
    Mem<char> d_xbuf;             // [flags: 64 x u32][hits: 8 x 3 x M x u64], IPC-exported
    PeerMem x_map[8], row_map[8]; // the other ranks' d_xbuf and d_row, mapped here
    void *x_peer[8] = {nullptr};  // (not owned) the same buffer of every rank (own: d_xbuf, others: x_map)
    int32_t *row_peer[8] = {nullptr};   // (not owned) every rank's can_see table (own: d_row, others: row_map)
    Mem<unsigned *> d_xflags2;    // device array of the ranks' barrier flag rows (xbuf + 128 bytes)
    unsigned xbar_count = 0;      // cross-GPU barriers issued so far (identical on every rank)
    Mem<unsigned> d_xstep;        // steps published so far (device-resident: the step count of a launch is data dependent)
    // per round
    Mem<int32_t> d_W, d_rem;
    int32_t *d_newc = nullptr;    // (not owned) right behind the scalars in d_scal
    Mem<u64> d_S;
    Mem<int8_t> d_famous;
    Mem<uint8_t> d_consensus, d_done, d_coin;
    Mem<i64> d_stake;
    Mem<int32_t> d_scal;
    // find_order
    Mem<int32_t> d_lastord, d_tx, d_idx, d_batch_ev, d_batch_seg, d_perm;
    int32_t *d_tx_rr = nullptr;   // (not owned) by order position, parallel to d_tx, in the same block
    double *d_tx_ts = nullptr;    // (not owned) likewise
    Mem<double> d_ts;
    Mem<u64> d_key;
    // find_order's per-round scratch, grown by order_scratch (d_seg_nf.cap() rounds)
    Mem<int32_t> d_seg_start, d_seg_fw, d_seg_nf, d_rounds_in, d_plan;
    Mem<uint8_t> d_seg_white;
    Mem<char> d_flush;
    // small appends (the reference's cadence: one sync per call): one packed copy instead of eight, from a ring of pinned
    // slots -- one view's columns (sw_append), or a batch's parameters and columns (sw_batch_append, on its first
    // engine).  h_vbuf cannot hold them: the batched fame and order calls of the same turn rewrite it on the host before
    // the asynchronous copy from it would have run.
    static constexpr int STAGE_SLOTS = 8, STAGE_EVENTS = 64;
    Pinned<uint8_t> h_stage;
    Mem<uint8_t> d_stage;         // STAGE_SLOTS slots of stage_bytes() each
    Event stage_ev[STAGE_SLOTS];
    int stage_next = 0;
    static constexpr int STREAM_N = 16;              // divide_rounds calls of at most this many events take the one-launch path
    Mem<StreamParams> d_stviews;                     // sw_batch_divide_rounds: the parameters of the views on that path
    Pinned<int32_t> h_scal;
    int32_t *h_newc = nullptr;    // (not owned) Rcap: right behind the scalars in h_scal (one copy brings both back)
    Event user_ev[16];
    std::vector<TimedSpan> spans;
    std::vector<Event> pool;      // timing events no span or append holds
    std::unordered_map<Id32, int32_t, Id32Hash> ids;     // sw_ingest: event id -> arrival index
    std::vector<Id32> id_of;                             // ... and back: arrival index -> id (zero: none), n_events or fewer
    // sw_sync_summary / sw_sync_reply (swirld_sync.cuh, owned by the first engine of a batch): the call's parameters,
    // tile starts and summaries go over in one copy from h_sync_in into d_sync, which also holds the tile scratch; the
    // kernels write their output straight into h_sync_out (pinned, so the device reaches it through unified addressing)
    Mem<char> d_sync;
    Pinned<char> h_sync_in, h_sync_out;
    // sw_verify_events (swirld_verify.cuh): the members' keys, libsodium's verdict on each key alone, [1..15](-A) per
    // member and [1..15]B; a call's inputs go over in one copy from h_vin, and its flags come back through h_vflags.
    // h_vkeys: the keys again on the host, where sw_batch_ingest_verified compares the views' keys
    bool have_keys = false, have_base = false;
    std::vector<uint8_t> h_vkeys;
    Mem<uint8_t> d_vkeys, d_vkey_ok;
    Mem<swv::gc> d_vatab, d_vbtab;
    Pinned<uint8_t> h_vin, h_vflags;
    Mem<uint8_t> d_vin, d_vk, d_vflags;
    // sw_set_signing_key / sw_new_events (swirld_sign.cuh): the comb table of j 256^k B, made once per engine; the
    // expanded key a || prefix || A of member sign_member, in device memory only (d_skin and h_skin stage libsodium's
    // secret key for one call and are wiped before it returns); a call's inputs go over through h_vin / d_vin, and its
    // signatures and ids come back through h_sout.
    bool have_sign = false, have_comb = false;
    int sign_member = -1;
    Mem<swv::gc> d_comb;
    Mem<uint8_t> d_sk, d_skin, d_sout;
    Pinned<uint8_t> h_skin, h_sout;
    sw_stats_t stats{};
    std::string err;
    size_t stage_bytes() const { return d_stage.cap() / STAGE_SLOTS; }
};

namespace {

int fail(sw_engine *e, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (e) e->err = buf; else g_create_error = buf;
    return code;
}

#define CK(call)                                                                         \
    do {                                                                                 \
        cudaError_t _s = (call);                                                         \
        if (_s != cudaSuccess)                                                           \
            return fail(e, SW_E_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(_s),   \
                        __FILE__, __LINE__);                                             \
    } while (0)

// call F<NJ>(args) for the engine's word count
#define SW_NJ(F, ...)                                                                    \
    (e->NJ == 1 ? F<1>(__VA_ARGS__) : e->NJ == 2 ? F<2>(__VA_ARGS__) : e->NJ == 4 ? F<4>(__VA_ARGS__) \
     : e->NJ == 8 ? F<8>(__VA_ARGS__) : e->NJ == 16 ? F<16>(__VA_ARGS__) : F<32>(__VA_ARGS__))

// call F<NC, UNIT>(args) for the M <= 64 kernels of engine x: its words per member set, and whether all stakes are 1
#define SW_NCU(x, F, ...)                                                                \
    ((x)->NC == 1 ? ((x)->unit ? F<1, true>(__VA_ARGS__) : F<1, false>(__VA_ARGS__))    \
                  : ((x)->unit ? F<2, true>(__VA_ARGS__) : F<2, false>(__VA_ARGS__)))

Event get_event(sw_engine *e) {                    // a timing event: one the pool has, or a new one
    Event ev;
    if (!e->pool.empty()) { ev = std::move(e->pool.back()); e->pool.pop_back(); }
    else ev.create(true);
    return ev;
}

// The time stream `st` takes from here to end(), or to the end of the scope: the one place timing events are recorded.
// The span owns its events (fold_spans returns them to the pool), except that a span inside another may borrow the
// other's start instead of recording its own (an event record costs the stream a few microseconds).
struct Span {
    sw_engine *e; cudaStream_t st; Event a, b; cudaEvent_t start; SpanCat cat;
    Span(sw_engine *e_, cudaStream_t st_, SpanCat cat_) : e(e_), st(st_), a(get_event(e_)), b(get_event(e_)), start(a.get()), cat(cat_) {
        cudaEventRecord(start, st);
    }
    // from the start of `outer`, on its stream: for what `outer` begins with
    Span(const Span &outer, SpanCat cat_) : e(outer.e), st(outer.st), b(get_event(outer.e)), start(outer.start), cat(cat_) {}
    void end() {
        if (!b.get()) return;
        cudaEventRecord(b.get(), st);
        e->spans.push_back(TimedSpan{start, std::move(a), std::move(b), cat});
    }
    ~Span() { end(); }
};

void fold_spans(sw_engine *e) {
    std::vector<TimedSpan> pending;
    for (auto &s : e->spans) {
        if (cudaEventQuery(s.b.get()) == cudaErrorNotReady) { pending.push_back(std::move(s)); continue; }   // (a scan still running on the copy stream)
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, s.a, s.b.get()) == cudaSuccess) {
            switch (s.cat) {
            case SpanCat::divide: e->stats.ms_divide_rounds += ms; break;
            case SpanCat::fame: e->stats.ms_decide_fame += ms; break;
            case SpanCat::order: e->stats.ms_find_order += ms; break;
            case SpanCat::scan: e->stats.ms_can_see += ms; e->stats.ms_divide_rounds += ms; break;
            case SpanCat::rounds: e->stats.ms_rounds_kernel += ms; break;
            case SpanCat::scan_in_divide: e->stats.ms_can_see += ms; break;
            }
        }
        if (s.own_a.get()) e->pool.push_back(std::move(s.own_a));
        e->pool.push_back(std::move(s.b));
    }
    e->spans.swap(pending);
}

// Make the compute stream wait for the appended batches that start below `upto` (all of them: upto < 0).
int wait_appends(sw_engine *e, int upto) {
    size_t k = 0;
    for (auto &a : e->appends) {
        if (upto >= 0 && a.base >= upto) { e->appends[k++] = std::move(a); continue; }
        CK(cudaStreamWaitEvent(e->stream.get(), a.done.get(), 0));
        e->pool.push_back(std::move(a.done));   // (re-recorded only after later work was enqueued behind the wait)
    }
    e->appends.resize(k);
    return 0;
}

// The streams `after` go on once everything stream `first` has been given so far has run: `ev` marks that point (one
// record, however many followers)
int follow(sw_engine *e, cudaStream_t first, const std::vector<cudaStream_t> &after, cudaEvent_t ev) {
    CK(cudaEventRecord(ev, first));
    for (cudaStream_t s : after) CK(cudaStreamWaitEvent(s, ev, 0));
    return 0;
}

// ... with an event borrowed from the pool of `e` (it is recorded again only after later work was queued behind the wait)
int follow(sw_engine *e, cudaStream_t first, cudaStream_t after) {
    Event ev = get_event(e);
    const int rc = follow(e, first, {after}, ev.get());
    e->pool.push_back(std::move(ev));
    return rc;
}

// every stream of the engine idle
int sync_streams(sw_engine *e) {
    for (const Stream *s : {&e->stream, &e->copy_stream, &e->rs.stream, &e->rs.prep})
        if (s->get()) CK(cudaStreamSynchronize(s->get()));
    return 0;
}

// A buffer and the elements grow() gives it
template <class T, bool P> struct Sized { Mem<T, P> &m; size_t n; };
template <class T, bool P> Sized<T, P> sized(Mem<T, P> &m, size_t n) { return {m, n}; }

// The one way a buffer grows.  Nothing happens while `need` <= `have` (in the caller's unit: events, rounds, views or
// bytes).  Else every stream of the engine goes idle, since a kernel or copy on any of them may still read the old
// buffers, and the buffers are freed and allocated again at the sizes the caller asks for; after a failure all of them
// are empty.  Grows are rare (most callers double), so the synchronisation stays off the steady state.
template <class... S>
int grow(sw_engine *e, size_t need, size_t have, S... bufs) {
    if (need <= have) return 0;
    if (sync_streams(e) < 0) return SW_E_CUDA;
    (bufs.m.reset(), ...);
    cudaError_t s = cudaSuccess;
    ((s = s == cudaSuccess ? bufs.m.alloc(bufs.n) : s), ...);
    if (s == cudaSuccess) return 0;
    (bufs.m.reset(), ...);
    return fail(e, SW_E_CUDA, "growing a buffer: %s", cudaGetErrorString(s));
}

int device_error(sw_engine *e) {     // after a sync: did a kernel flag an error?
    int code = e->h_scal.get()[SC_ERR];
    if (code < 0) {
        const char *what = code == SW_E_CAPACITY ? "round table exhausted"
                         : code == SW_E_INDEX ? "list index out of range (swirld.py:305: a single seer)"
                         : code == SW_E_KEY ? "KeyError (undecided witness in a consensus round)"
                         : code == SW_E_CUDA ? "an exchange inside the round kernel timed out (a peer GPU, or a CTA of the cluster kernel, did not publish its step)" : "device error";
        return fail(e, code, "%s", what);
    }
    return 0;
}

// Everything but the ahead path writes the engine's own Wf, ring and counts: before it runs, the compute stream waits for
// the round stream's piece, which is given up (its rounds are computed again), and so are the round stream's copies.
// (The round stream runs its pieces in order: waiting for the end of the last one waits for all of them.)  This is the
// one way the round stream's state is given up: after it the stream holds nothing and its copies are not valid.
// `keys`: the caller clears the mask cache as well (reset_state), so the launch numbers that key it start again; at any
// other time a number used before could match a mask cached by that launch.
int rs_drain(sw_engine *e, bool keys = false) {
    RoundStream &rs = e->rs;
    const cudaEvent_t last = rs.pieces.empty() ? rs.tail.get() : rs.pieces.back().done.get();
    if (rs.synced && last) CK(cudaStreamWaitEvent(e->stream.get(), last, 0));
    rs.synced = false;
    for (auto &p : rs.pieces) rs.free.push_back(std::move(p.done));
    rs.pieces.clear();
    if (rs.tail.get()) rs.free.push_back(std::move(rs.tail));
    if (keys) rs.epoch = 0;
    return 0;
}

// Everything back to no events divided (and none appended, unless `keep_events`), once what is queued has run
int reset_state(sw_engine *e, bool keep_events = false) {
    if (wait_appends(e, -1) < 0 || rs_drain(e, true) < 0) return SW_E_CUDA;      // (true: the mask cache is cleared below)
    CK(cudaStreamSynchronize(e->stream.get()));
    fold_spans(e);
    const size_t RM = (size_t)e->Rcap * e->M;
    k_fill_i32<<<256, 256, 0, e->stream.get()>>>(e->d_W.get(), -1, RM);
    CK(cudaMemsetAsync(e->d_famous.get(), 0xff, RM, e->stream.get()));
    CK(cudaMemsetAsync(e->d_consensus.get(), 0, e->Rcap, e->stream.get()));
    CK(cudaMemsetAsync(e->d_famous_ev.get(), 0xff, e->cap, e->stream.get()));
    k_fill_i32<<<256, 256, 0, e->stream.get()>>>(e->d_idx.get(), -1, (size_t)e->cap);
    k_fill_i32<<<4, 256, 0, e->stream.get()>>>(e->d_lastord.get(), -1, (size_t)e->MP);
    k_fill_i32<<<4, 256, 0, e->stream.get()>>>(e->d_cs_carry.get(), -1, (size_t)e->MP);
    k_fill_i32<<<256, 256, 0, e->stream.get()>>>(e->d_Wf.get(), -1, RM);
    CK(cudaMemsetAsync(e->d_rbtot.get(), 0, sizeof(int32_t) * e->MP, e->stream.get()));
    k_fill_i32<<<64, 256, 0, e->stream.get()>>>(e->d_gchain.get(), -1, (size_t)e->MP * RB_RING);
    if (e->wide) {
        CK(cudaMemsetAsync(e->d_Sw.get(), 0, RM * e->NJ * sizeof(unsigned), e->stream.get()));
        CK(cudaMemsetAsync(e->d_sctag.get(), 0, sizeof(u64) * (size_t)e->cap, e->stream.get()));
    } else {
        CK(cudaMemsetAsync(e->d_S.get(), 0, RM * sizeof(u64), e->stream.get()));
        CK(cudaMemsetAsync(e->d_sc.get(), 0, sizeof(ulonglong2) * (size_t)e->cap, e->stream.get()));
    }
    int32_t sc[SC_COUNT] = {0};
    sc[SC_MAX_ROUND] = -1;
    CK(cudaMemcpyAsync(e->d_scal.get(), sc, sizeof sc, cudaMemcpyHostToDevice, e->stream.get()));
    CK(cudaStreamSynchronize(e->stream.get()));
    e->stats.kernel_launches += 5;
    e->n_divided = e->n_tx = 0;
    e->n_rowed = 0;
    e->rb_epoch = 0;
    if (!keep_events) {
        e->n_events = 0;
        std::fill(e->h_head.begin(), e->h_head.end(), -1);
        std::fill(e->h_count.begin(), e->h_count.end(), 0);
        e->snap_at.clear(); e->snap_cnt.clear(); e->snap_kept = 0;
    }
    memset(e->h_scal.get(), 0, sizeof(int32_t) * SC_COUNT);
    return 0;
}

// blocks of the scan of [first, first+n) (n > 24), of *B events each
int cs_blocks(const sw_engine *e, int first, int n, int *B_out) {
    // block length: >= 16 (32 above 64 members) events per member and block, so that nearly every member's last event of a
    // block sees every block-start head (then the finality check passes; the rest goes through the waves)
    int B = std::max(e->cs_min_B, std::min((e->M <= 64 ? 16 : 32) * e->M, 1 << 15));      // (above 64 members seeing every head takes more events per member)
    B = (B + 3) & ~3;
    const int first_al = first & ~3;
    int nb = (first + n <= first_al + B) ? 1 : 1 + (first + n - (first_al + B) + B - 1) / B;
    if (nb > 1 && first + n - (first_al + (nb - 1) * B) < 3 * B / 4) nb--;     // a short tail joins the block before it
    *B_out = B;
    return nb;
}

// the launches of the scan of [first, first+n)
int cs_launches(const sw_engine *e, int first, int n) {
    int B;
    return n <= 0 ? 0 : n <= 24 ? 1 : cs_blocks(e, first, n, &B) > 1 ? 9 : 4;
}

// can_see rows of the appended events [n_rowed, upto): the column-tiled blocked scan of swirld_cansee.cuh.
// `st`: the compute stream (lazily, from sw_divide_rounds) or the copy stream (eagerly, from sw_append: the
// scan of a new chunk then runs beside the round kernel of the previous one).  The two never overlap: a scan
// on one stream first waits for the last scan issued on the other (they share the scratch and the carry heads).
// `cat`: the span category of its time (fold_spans).
int cansee_scan(sw_engine *e, cudaStream_t st, int upto, SpanCat cat = SpanCat::scan) {
    const int first = e->n_rowed, n = upto - e->n_rowed;
    if (n <= 0) return 0;
    const int M = e->M;
    CsParams C{};
    C.M = M; C.first = first; C.n = n;
    C.p0 = e->d_p0.get(); C.p1 = e->d_p1.get(); C.creator = e->d_creator.get(); C.stale = e->d_stale.get(); C.row = e->d_row.get();
    C.meta = e->d_cs_meta.get(); C.wr = e->d_cs_wr.get(); C.xb = e->d_cs_xb.get(); C.last = e->d_cs_last.get(); C.Qtab = e->d_cs_Q.get();
    C.carry = e->d_cs_carry.get(); C.slow_list = e->d_cs_slow.get(); C.slow_cnt = e->d_cs_slowcnt.get(); C.sflag = e->d_cs_sflag.get(); C.xlist = e->d_cs_xlist.get(); C.slow_blk = e->d_cs_slowblk.get(); C.blk_cnt = e->d_cs_blkcnt.get();
    if (n <= 24) {                                     // the reference's own cadence: a handful of events per call
        {
            Span sp(e, st, cat);
            k_cs_small<<<1, std::min(1024, (M + 31) / 32 * 32), 0, st>>>(C);
        }
        CK(cudaGetLastError());
        e->stats.kernel_launches += 1;
        e->n_rowed = upto;
        return 0;
    }
    int B;
    C.nb = cs_blocks(e, first, n, &B);
    C.B = B;
    C.first_al = first & ~3;
    // columns per tile: 32 (one warp = one 128-byte row segment) unless the per-member cache val[M][CT] then limits a
    // SM to so few CTAs that narrower tiles finish in fewer waves (M = 1024: 128 KB per CTA at CT = 32)
    const bool has_stale = e->h_stale_cum[first + n] - e->h_stale_cum[first] > 0;
    C.SV = has_stale ? CS_SV : 0;
    int CT = 32;
    {
        long long best = -1;
        for (int ct = 32; ct >= 8; ct >>= 1) {
            const long long smem_ct = (long long)(M + C.SV) * ct * 4 + CS_TILE * 16 + 3 * CS_TILE;
            const long long conc = std::max(1LL, std::min(32LL, (220LL << 10) / smem_ct));
            const long long ctas = (long long)C.nb * ((M + ct - 1) / ct);
            const long long waves = (ctas + e->n_sm * conc - 1) / (e->n_sm * conc);
            if (best < 0 || waves < best) { best = waves; CT = ct; }
        }
    }
    C.CT = CT;
    int tile_lo = 0, tile_hi = (M + CT - 1) / CT;
    const bool shard = e->nranks > 1;
    if (shard) {                                          // the column tiles of this rank; every rank stores into every table
        const int nt = tile_hi;
        tile_lo = (int)((long long)nt * e->rank / e->nranks); tile_hi = (int)((long long)nt * (e->rank + 1) / e->nranks);
        C.npeer = e->nranks;
        for (int p = 0; p < e->nranks; p++) C.prow[p] = e->row_peer[p];
    }
    C.tile_lo = tile_lo;
    const int ntiles = std::max(0, tile_hi - tile_lo);
    auto xbarrier = [&]() -> int {
        if (!shard) return 0;
        k_xbarrier<<<1, 32, 0, st>>>(e->d_xflags2.get(), e->rank, e->nranks, ++e->xbar_count, e->d_scal.get());
        CK(cudaGetLastError());
        return 0;
    };
    const size_t smem = (size_t)(M + C.SV) * CT * sizeof(int) + CS_TILE * sizeof(int4) + 3 * CS_TILE;
    const int pblocks = std::max(1, std::min(8 * e->n_sm, (n + 255) / 256));
    k_fill_i32<<<std::max(1, std::min(256, (int)(((size_t)C.nb * M + 255) / 256))), 256, 0, st>>>(e->d_cs_last.get(), -1, (size_t)C.nb * M);
    if (C.nb > 1) {
        CK(cudaMemsetAsync(e->d_cs_wr.get() + first, 0, (size_t)n, st));
        CK(cudaMemsetAsync(e->d_cs_xb.get() + (first & ~3), 0, (size_t)(n + (first & 3)), st));
        CK(cudaMemsetAsync(e->d_cs_sflag.get() + first, 0, (size_t)n, st));
        CK(cudaMemsetAsync(e->d_cs_slowcnt.get(), 0, sizeof(int32_t) * 4, st));
        CK(cudaMemsetAsync(e->d_cs_blkcnt.get(), 0, sizeof(int32_t) * (size_t)C.nb, st));
    }
    Span sp(e, st, cat);
    k_cs_prep<<<pblocks, 256, 0, st>>>(C);
    if (C.nb > 1) {
        if (ntiles > 0) {
            const dim3 g(C.nb, ntiles);
            if (shard) { if (has_stale) k_cs_pass<1, true, true><<<g, CS_CT, smem, st>>>(C); else k_cs_pass<1, false, true><<<g, CS_CT, smem, st>>>(C); }
            else { if (has_stale) k_cs_pass<1, true, false><<<g, CS_CT, smem, st>>>(C); else k_cs_pass<1, false, false><<<g, CS_CT, smem, st>>>(C); }
        }
        if (xbarrier() < 0) return SW_E_CUDA;              // every rank's partial rows are in every table
    }
    k_cs_heads<<<std::max(1, std::min(2 * e->n_sm, (int)(((size_t)(C.nb + 1) * M + 255) / 256))), 256, 0, st>>>(C);
    if (C.nb > 1) {
        k_cs_check<<<std::max(1, std::min(4 * e->n_sm, (int)(((size_t)C.nb * M + 7) / 8))), 256, 0, st>>>(C);
        const size_t ssm = (size_t)CS_SLOW_WARPS * M * sizeof(int);
        k_cs_slow_wave<<<e->n_sm, CS_SLOW_WARPS * 32, ssm, st>>>(C, 1);
        k_cs_slow_wave<<<e->n_sm, CS_SLOW_WARPS * 32, ssm, st>>>(C, 2);
        k_cs_slow_rest<<<1, CS_REST_WARPS * 32, (size_t)CS_REST_WARPS * M * sizeof(int), st>>>(C);
    }
    if (ntiles > 0) {
        const dim3 g(C.nb, ntiles);
        if (shard) { if (has_stale) k_cs_pass<2, true, true><<<g, CS_CT, smem, st>>>(C); else k_cs_pass<2, false, true><<<g, CS_CT, smem, st>>>(C); }
        else { if (has_stale) k_cs_pass<2, true, false><<<g, CS_CT, smem, st>>>(C); else k_cs_pass<2, false, false><<<g, CS_CT, smem, st>>>(C); }
    }
    if (shard) k_cs_carry<<<(M + 255) / 256, 256, 0, st>>>(C);
    if (xbarrier() < 0) return SW_E_CUDA;                  // the whole table is in every rank's memory
    sp.end();
    CK(cudaGetLastError());
    e->stats.kernel_launches += C.nb > 1 ? 9 : 4;
    e->n_rowed = upto;
    return 0;
}

void push_snapshot(sw_engine *e, int at, const std::vector<int32_t> &cnt) {
    e->snap_at.push_back(at);
    e->snap_cnt.insert(e->snap_cnt.end(), cnt.begin(), cnt.end());
}

// the snapshot at the end of an append.  The earlier end-of-append ones below n_divided go first: divides only go
// forward, and after sw_rewind the SNAP-event ones keep counts_at exact.  So snapshots cost memory per event, not per
// append (4 KB per append at M = 1024 otherwise).
void push_append_snapshot(sw_engine *e) {
    if (!e->snap_at.empty() && e->snap_at.back() == e->n_events) return;     // (the append ended on a SNAP-event one)
    const int M = e->M;
    size_t k = e->snap_kept, i = k;
    for (; i < e->snap_at.size() && e->snap_at[i] < e->n_divided; i++)
        if (e->snap_at[i] % sw_engine::SNAP == 0) {
            e->snap_at[k] = e->snap_at[i];
            std::copy_n(e->snap_cnt.begin() + i * M, M, e->snap_cnt.begin() + k * M);
            k++;
        }
    e->snap_at.erase(e->snap_at.begin() + k, e->snap_at.begin() + i);
    e->snap_cnt.erase(e->snap_cnt.begin() + k * M, e->snap_cnt.begin() + i * M);
    e->snap_kept = k;
    push_snapshot(e, e->n_events, e->h_count);
}

// events of each member among the first x appended events: the nearest snapshot at or below x, then the rest one by one
void counts_at(const sw_engine *e, int x, int32_t *out) {
    const int M = e->M;
    const auto it = std::upper_bound(e->snap_at.begin(), e->snap_at.end(), x);
    int from = 0;
    if (it == e->snap_at.begin()) std::fill(out, out + M, 0);
    else {
        const size_t k = (size_t)(it - e->snap_at.begin()) - 1;
        from = e->snap_at[k];
        std::copy_n(e->snap_cnt.begin() + k * M, M, out);
    }
    for (int i = from; i < x; i++) out[e->h_creator[i]]++;
}

// A chunk meta block, one layout for both kernel families (MP = max(M, 64) members): d_rbmeta of the compute stream
// and the round stream's two blocks (RoundStream::meta), rb_meta_ints(MP) ints each
struct RbMeta {
    int32_t *ccnt, *cmin, *coff;  // [MP], [MP], [MP + 1]: the chunk's per-member counts, smallest seqs, offsets (k_rb_prep)
    unsigned *bar;                // grid barrier counter of the round kernel
    int32_t *wcnt;                // [2] witnesses of the chunk (k_rb_finish; the ahead path alternates, RoundStream::wslot)
    unsigned *ticket;             // [3] k_rounds_wide's work counters
    int32_t *ctot;                // [MP] the round stream's per-member counts at the end of its piece (the compute
                                  // stream keeps its own in d_rbtot)
};

size_t rb_meta_ints(int MP) { return 4 * (size_t)MP + 64; }

RbMeta rb_meta(int32_t *m, int MP) {
    return RbMeta{m, m + MP, m + 2 * MP, reinterpret_cast<unsigned *>(m + 3 * MP + 8), m + 3 * MP + 9,
                  reinterpret_cast<unsigned *>(m + 3 * MP + 12), m + 3 * MP + 16};
}

// What the kernels of a chunk keep from chunk to chunk, and the chunk's scratch: the engine's own, which is what a
// caller sees, or the round stream's for its buffers b (RoundStream).  `rsg`: the cluster kernel's seq-space rows.
struct RoundTarget { RbMeta meta; int32_t *Wf, *gchain, *ctot, *scal, *rsg; };

RoundTarget own_target(const sw_engine *e) {
    return {rb_meta(e->d_rbmeta.get(), e->MP), e->d_Wf.get(), e->d_gchain.get(), e->d_rbtot.get(), e->d_scal.get(), e->d_rsg[0].get()};
}

RoundTarget rs_target(const sw_engine *e, int b) {
    const RbMeta m = rb_meta(e->rs.meta.get() + b * rb_meta_ints(e->MP), e->MP);
    return {m, e->rs.Wf.get(), e->rs.gchain.get(), m.ctot, e->rs.scal.get(), e->d_rsg[b].get()};
}

// what both kernel families read of the round-batch parameters: the chunk, its grouping by creator (k_rb_prep) and
// the pass after the round kernel (k_rb_finish)
RbParams chunk_params(const sw_engine *e, const RoundTarget &T, int first, int n) {
    RbParams R{};
    R.M = e->M; R.first = first; R.n = n; R.Rcap = e->Rcap;
    R.row = e->d_row.get(); R.p0 = e->d_p0.get(); R.creator = e->d_creator.get(); R.seq = e->d_seq.get(); R.round = e->d_round.get();
    R.cev = e->d_cev.get(); R.ctot = T.ctot; R.gchain = T.gchain; R.wit = e->d_wit.get(); R.W = e->d_W.get();
    R.ccnt = T.meta.ccnt; R.cmin = T.meta.cmin; R.coff = T.meta.coff; R.bar = T.meta.bar; R.wcnt = T.meta.wcnt;
    R.wlist = e->d_cev.get() + e->cap;
    return R;
}

// the chunk's events grouped by creator (k_rb_prep) from the per-member counts of the host mirror: [first, first+n)
// holds seqs [lo[c], hi[c]) of member c.  `rsg` (M <= 64): also the seq-space rows of the cluster round kernel.
template <int CM>
int chunk_prep(sw_engine *e, const RbParams &R, int32_t *rsg, cudaStream_t st) {
    RbChunk<CM> K;
    int32_t lo[CM];
    counts_at(e, R.first, lo);
    counts_at(e, R.first + R.n, K.ctot);
    int o = 0;
    for (int c = 0; c < CM; c++) {
        const int cnt = c < e->M ? K.ctot[c] - lo[c] : 0;
        K.ccnt[c] = cnt; K.cmin[c] = cnt > 0 ? lo[c] : 0x7f7f7f7f;
        if (c >= e->M) K.ctot[c] = 0;
        K.coff[c] = o; o += cnt;
    }
    K.coff[CM] = o;
    k_rb_prep<CM><<<std::max(1, std::min(8 * e->n_sm, (R.n + 7) / 8)), 256, 0, st>>>(R, K, rsg);
    CK(cudaGetLastError());
    return 0;
}

// what the round kernels read besides the chunk: Wf and the scalars of the target, launch number `epoch`
RbParams round_params(const sw_engine *e, const RoundTarget &T, int first, int n, int grid, int min_L, unsigned epoch) {
    RbParams R = chunk_params(e, T, first, n);
    R.L = std::max(std::min(min_L, RB_LMAX), std::min(RB_LMAX, grid * (RB_THREADS / 32) / e->M));
    R.Wf = T.Wf; R.sc = e->d_sc.get();
    R.res = e->d_res.get(); R.stake = e->d_stake.get(); R.tot2 = 2 * e->tot; R.scal = T.scal;
    R.SM = e->d_SM.get(); R.dbg = e->d_dbg.get();
    R.epoch = epoch;
    return R;
}

// The chunk goes to the cluster round kernel first: its parameters, with the seq-space rows of the target; the
// cooperative kernel's R then continues from where the cluster stopped
RcParams cluster_first(const sw_engine *e, const RoundTarget &T, RbParams &R) {
    const RcParams Q{R, T.rsg, e->d_rccont.get(), e->d_rcslog.get()};
    R.cont = e->d_rccont.get();
    return Q;
}

// CTAs of one view's round kernels: 16 SMs stay free for the can_see scan of the next chunk
int round_grid(const sw_engine *e) { return std::max(e->n_sm / 2, e->n_sm - 16); }

// buffer b of the cluster kernel's seq-space rows, for n events
int rsg_reserve(sw_engine *e, int n, int b = 0) {
    const size_t want = std::min<size_t>((size_t)e->cap, std::max<size_t>((size_t)n, 1 << 16));
    return grow(e, n, e->d_rsg[b].cap() / 64, sized(e->d_rsg[b], want * 64));
}

// rounds of the chunk by the cooperative round-batch kernel (swirld_rounds.cuh), M <= 64: parameters R + the grouping
// of the chunk (`grid` = CTAs this view's round kernel will run on).  `rc`: the chunk goes to the cluster round kernel
// first, with the parameters Q.
int round_batch_prep(sw_engine *e, int first, int n, int grid, int min_L, bool rc, RbParams &R, RcParams &Q) {
    if (rc && rsg_reserve(e, n) < 0) return SW_E_CUDA;
    const RoundTarget T = own_target(e);
    R = round_params(e, T, first, n, grid, min_L, ++e->rb_epoch);
    if (chunk_prep<64>(e, R, rc ? T.rsg : nullptr, e->stream.get()) < 0) return SW_E_CUDA;
    e->stats.kernel_launches += 1;
    if (rc) Q = cluster_first(e, T, R);
    return 0;
}

// what follows the round kernel: ring of recent events, witness flags / table / list, seen-masks, strongly-seen sets
template <int NC>
int round_batch_finish(sw_engine *e, const RbParams &R, const RbFold &F = RbFold{}) {
    const int n = R.n, blocks = std::max(1, std::min(296, (n + 255) / 256));
    k_rb_finish<<<blocks, 256, 0, e->stream.get()>>>(R, F);
    k_rb_seenmask<NC><<<(n + 7) / 8, 256, 0, e->stream.get()>>>(R);
    CK(cudaGetLastError());
    StrongParams Q{};
    Q.M = e->M; Q.first = R.first; Q.n = n; Q.Rcap = e->Rcap; Q.creator = e->d_creator.get(); Q.row = e->d_row.get();
    Q.round = e->d_round.get(); Q.wit = e->d_wit.get(); Q.SM = e->d_SM.get(); Q.S = e->d_S.get(); Q.stake = e->d_stake.get(); Q.tot2 = 2 * e->tot;
    Q.coin = e->d_coin.get(); Q.sig = e->d_sig.get(); Q.unit = e->unit ? 1 : 0;
    Q.list = R.wlist; Q.list_n = R.wcnt;
    const int sblocks = std::max(1, std::min((n + 7) / 8, 4 * e->n_sm));
    k_strong<NC><<<sblocks, 256, 0, e->stream.get()>>>(Q);
    CK(cudaGetLastError());
    e->stats.kernel_launches += 3;
    return 0;
}

// one thread-block cluster per view (blockIdx.y)
void rc_launch_config(cudaLaunchConfig_t &cfg, cudaLaunchAttribute *at, int clusters, cudaStream_t stream) {
    cfg = cudaLaunchConfig_t{};
    cfg.gridDim = dim3(RC_CS, clusters); cfg.blockDim = dim3(RC_THREADS); cfg.dynamicSmemBytes = RC_SMEM_BYTES; cfg.stream = stream;
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = RC_CS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
}

// sw_create: the cluster round kernel's launch attributes, and how many of its clusters the device holds at once
template <int NC, bool UNIT>
cudaError_t rc_setup(int *clusters) {
    cudaError_t er = cudaSuccess;
    for (const void *fn : {(const void *)k_rounds_cluster<UNIT, RcParams>, (const void *)k_rounds_cluster<UNIT, const RcParams *>,
                           (const void *)k_rounds_cluster_log<UNIT>}) {
        if (er == cudaSuccess) er = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RC_SMEM_BYTES);
        if (er == cudaSuccess) er = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    }
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at[1];
    rc_launch_config(cfg, at, 1, nullptr);
    if (er == cudaSuccess) er = cudaOccupancyMaxActiveClusters(clusters, (const void *)k_rounds_cluster<UNIT, const RcParams *>, &cfg);
    return er;
}

// The round kernels of nv views' chunks on stream `st`, G CTAs per view: with `rc` the chunk inside one thread-block
// cluster per view first, then the cooperative kernel, which takes over whatever a cluster hands back (normally nothing).
// R and Q are one view's parameters (nv = 1) or the device arrays of nv views'.
template <int NC, bool UNIT, class RSrc, class QSrc>
int round_kernels(sw_engine *e, RSrc R, QSrc Q, int nv, int G, bool rc, cudaStream_t st) {
    if (rc) {
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute at[1];
        rc_launch_config(cfg, at, nv, st);
        if constexpr (std::is_same<QSrc, RcParams>::value) {
            if (Q.slog) CK(cudaLaunchKernelEx(&cfg, k_rounds_cluster_log<UNIT>, Q));    // (SW_RC_STEPS)
            else CK(cudaLaunchKernelEx(&cfg, k_rounds_cluster<UNIT, QSrc>, Q));
        } else CK(cudaLaunchKernelEx(&cfg, k_rounds_cluster<UNIT, QSrc>, Q));
    }
    void *args[] = {(void *)&R};
    CK(cudaLaunchCooperativeKernel((void *)k_rounds_batch<NC, UNIT, RSrc>, dim3(G, nv), dim3(RB_THREADS), args, 0, st));
    return 0;
}

// what the round kernels of one call count, wherever they ran
void count_round_kernels(sw_engine *e, bool rc) {
    e->stats.kernel_launches += rc ? 2 : 1;
    e->stats.rounds_cluster_launches += rc ? 1 : 0;
}

// `call`: the caller's span, opened just before: the round kernels' span starts with it
template <int NC, bool UNIT>
int divide_round_batch(sw_engine *e, int first, int n, const Span &call) {
    const int grid = round_grid(e);
    const bool rc = e->rc_ok && n >= e->rc_min_n;
    RbParams R;
    RcParams Q{};
    {
        Span sp(call, SpanCat::rounds);
        if (round_batch_prep(e, first, n, grid, 1, rc, R, Q) < 0 || round_kernels<NC, UNIT>(e, R, Q, 1, grid, rc, e->stream.get()) < 0)
            return SW_E_CUDA;
        count_round_kernels(e, rc);
    }
    return round_batch_finish<NC>(e, R);
}

// ---- the rounds run ahead (RoundStream)
int rs_create(sw_engine *e) {
    RoundStream &rs = e->rs;
    const size_t RM = (size_t)e->Rcap * e->M;
    CK(rs.stream.create()); CK(rs.prep.create()); CK(rs.wait.create());
    for (int b = 0; b < 2; b++) { CK(rs.prepped[b].create()); CK(rs.bufdone[b].create()); }
    CK(rs.Wf.alloc(RM)); CK(rs.gchain.alloc((size_t)e->MP * RB_RING));
    CK(rs.meta.alloc(2 * rb_meta_ints(e->MP))); CK(rs.scal.alloc(SC_COUNT));
    rs.on = true;
    return 0;
}

// the round stream and its prep stream go on after what the compute stream has been given so far
int rs_follow(sw_engine *e) { return follow(e, e->stream.get(), {e->rs.stream.get(), e->rs.prep.get()}, e->rs.wait.get()); }

// the round stream's copies of the engine's Wf, ring and scalars, at the first call of a run of ahead calls
int rs_sync(sw_engine *e) {
    RoundStream &rs = e->rs;
    if (rs.synced) return 0;
    if (rs_follow(e) < 0) return SW_E_CUDA;
    CK(cudaMemcpyAsync(rs.Wf.get(), e->d_Wf.get(), sizeof(int32_t) * e->Rcap * e->M, cudaMemcpyDeviceToDevice, rs.stream.get()));
    CK(cudaMemcpyAsync(rs.gchain.get(), e->d_gchain.get(), sizeof(int32_t) * e->MP * RB_RING, cudaMemcpyDeviceToDevice, rs.stream.get()));
    CK(cudaMemcpyAsync(rs.scal.get(), e->d_scal.get(), sizeof(int32_t) * SC_COUNT, cudaMemcpyDeviceToDevice, rs.stream.get()));
    CK(cudaMemsetAsync(rb_meta(e->d_rbmeta.get(), e->MP).wcnt, 0, 2 * sizeof(int32_t), e->stream.get()));
    rs.wslot = 0;
    rs.rounded = e->n_divided;
    rs.synced = true;
    return 0;
}

// Rounds of [first, first+n) on the round stream's target, in the order RoundStream states.  The caller has made the
// prep stream wait for the piece's rows.  k_rb_prep runs there; then on the round stream, after the prep,
// k_rounds_cluster and the hand-over launch of k_rounds_batch, the piece's end, and last the ring update.
template <int NC, bool UNIT>
int rs_piece(sw_engine *e, int first, int n) {
    RoundStream &rs = e->rs;
    const int b = rs.buf;
    rs.buf ^= 1;
    if (rsg_reserve(e, n, b) < 0) return SW_E_CUDA;
    const int grid = round_grid(e);
    const RoundTarget T = rs_target(e, b);
    RbParams R = round_params(e, T, first, n, grid, 1, 0x80000000u | ++rs.epoch);
    CK(cudaStreamWaitEvent(rs.prep.get(), rs.bufdone[b].get(), 0));
    if (chunk_prep<64>(e, R, T.rsg, rs.prep.get()) < 0) return SW_E_CUDA;
    if (follow(e, rs.prep.get(), {rs.stream.get()}, rs.prepped[b].get()) < 0) return SW_E_CUDA;
    const RcParams Q = cluster_first(e, T, R);
    if (round_kernels<NC, UNIT>(e, R, Q, 1, grid, true, rs.stream.get()) < 0) return SW_E_CUDA;
    CK(cudaEventRecord(rs.bufdone[b].get(), rs.stream.get()));
    if (rs.tail.get()) rs.free.push_back(std::move(rs.tail));      // (the piece that ended there is the last one no more)
    Event done;
    if (!rs.free.empty()) { done = std::move(rs.free.back()); rs.free.pop_back(); }
    else CK(done.create());
    CK(cudaEventRecord(done.get(), rs.stream.get()));
    rs.pieces.push_back({first + n, std::move(done)});
    RbRing G;
    G.ring = T.gchain; G.creator = e->d_creator.get(); G.seq = e->d_seq.get(); G.rfirst = first; G.rn = n;
    counts_at(e, first + n, G.ctot);
    k_rb_ring<<<std::max(1, std::min(2 * e->n_sm, (n + 255) / 256)), 256, 0, rs.stream.get()>>>(G);
    CK(cudaGetLastError());
    rs.rounded = first + n;
    return 0;
}

bool ahead_path(const sw_engine *e, int n) { return e->rs.on && !e->wide && e->rc_ok && n >= e->rc_min_n && e->nranks == 1; }

// A piece queued ahead covers up to RS_CALLS call lengths of rows, and half the rows left at most, so that near the end
// of the rows the pieces shrink back to one call: every call after the last piece would wait for all of that piece's
// rounds before its finish and fame kernels could run.
constexpr int RS_CALLS = 8;

// the last can_see rows were written on the compute stream: a scan on the copy stream waits for them
int rows_written(sw_engine *e) {
    CK(cudaEventRecord(e->scan_ev.get(), e->stream.get()));
    e->scan_ev_set = true;
    return 0;
}

int rs_ahead_len(const sw_engine *e, int n) {
    const int avail = e->n_rowed - e->rs.rounded;
    return std::min(avail, n * std::max(1, std::min(RS_CALLS, avail / n / 2)));
}

// sw_divide_rounds on the ahead path.  The call's rounds come from the round stream: a piece for whatever part of
// [first, first+n) none covers yet, then the compute stream waits for the piece that holds the call's end.  The finish
// kernels publish the call's part of the round stream's state (RbFold).  While the can_see rows reach beyond the pieces,
// more start on the round stream behind them, until two end beyond this call, so that the round stream is never idle
// waiting for a call.  The call counts the launches and the launch number (rb_epoch) the same call makes without the
// round stream, so the counters do not depend on where pieces begin.  `scan_from` >= 0: the call scanned only its own
// rows, from there (sw_divide_rounds); the rest are scanned here, beside the call's piece, and charged as one scan.
template <int NC, bool UNIT>
int divide_ahead(sw_engine *e, int first, int n, int scan_from) {
    RoundStream &rs = e->rs;
    const int end = first + n;
    if (rs_sync(e) < 0) return SW_E_CUDA;
    const bool cover = rs.rounded < end;
    if (cover && (rs_follow(e) < 0 || rs_piece<NC, UNIT>(e, rs.rounded, end - rs.rounded) < 0))
        return SW_E_CUDA;
    if (scan_from >= 0) {
        // (after the piece's k_rb_prep: its cluster kernel is then the first to claim the SMs the prep frees, and the
        //  scan takes what the cluster leaves)
        if (cover) CK(cudaStreamWaitEvent(e->stream.get(), rs.prepped[rs.buf ^ 1].get(), 0));
        const i64 kl = e->stats.kernel_launches;
        if (cansee_scan(e, e->stream.get(), e->n_events, SpanCat::scan_in_divide) < 0 || rows_written(e) < 0) return SW_E_CUDA;
        e->stats.kernel_launches = kl + cs_launches(e, scan_from, e->n_events - scan_from) - cs_launches(e, scan_from, end - scan_from);
    }
    // (the pieces are contiguous from n_divided and the last ends at `rounded` >= end: one of them holds the call's end)
    size_t k = 0;
    while (k + 1 < rs.pieces.size() && rs.pieces[k].end < end) k++;
    if (rs.pieces.empty() || rs.pieces[k].end < end) return fail(e, SW_E_CUDA, "divide_ahead: no piece holds the call's end");
    CK(cudaStreamWaitEvent(e->stream.get(), rs.pieces[k].done.get(), 0));
    if (rs.pieces[k].end == end) k++;
    // the pieces the call has waited for leave the queue; the end of the last piece of all stays findable (rs_drain)
    if (k == rs.pieces.size()) { rs.tail = std::move(rs.pieces.back().done); k--; rs.pieces.pop_back(); }
    for (size_t i = 0; i < k; i++) rs.free.push_back(std::move(rs.pieces[i].done));
    rs.pieces.erase(rs.pieces.begin(), rs.pieces.begin() + k);
    const RoundTarget T = own_target(e);
    RbParams R = chunk_params(e, T, first, n);
    R.SM = e->d_SM.get(); R.wcnt = T.meta.wcnt + rs.wslot;
    RbFold F{};
    F.on = 1; F.Wf = T.Wf; F.scal = T.scal; F.wnext = T.meta.wcnt + (rs.wslot ^ 1); F.rscal = rs.scal.get();
    counts_at(e, end, F.ctot);
    rs.wslot ^= 1;
    e->rb_epoch++;
    e->stats.kernel_launches += 1;                      // (k_rb_prep)
    count_round_kernels(e, true);
    if (round_batch_finish<NC>(e, R, F) < 0) return SW_E_CUDA;
    while (rs.pieces.size() < 2) {
        const int len = rs_ahead_len(e, n), next = rs.rounded + len;
        if (len < e->rc_min_n) break;
        for (auto &a : e->appends) if (a.base < next) CK(cudaStreamWaitEvent(rs.prep.get(), a.done.get(), 0));
        if (e->scan_ev_set) CK(cudaStreamWaitEvent(rs.prep.get(), e->scan_ev.get(), 0));
        if (rs_piece<NC, UNIT>(e, rs.rounded, len) < 0) return SW_E_CUDA;
    }
    return 0;
}

size_t rounds_wide_smem(int M) { return (size_t)(2 * M + 16 * M + 1 + 32 + (RW_THREADS / 32) * M + 1) * sizeof(int); }

// rounds of the chunk for any member count (swirld_wide.cuh)
template <int NJ>
int divide_rounds_wide(sw_engine *e, int first, int n) {
    const int M = e->M;
    const RbParams T = chunk_params(e, own_target(e), first, n);    // the grouping and the finish kernel shared with the M <= 64 path
    if (chunk_prep<SW_MAX_MEMBERS>(e, T, nullptr, e->stream.get()) < 0) return SW_E_CUDA;
    e->stats.kernel_launches += 1;
    RwParams R{};
    R.M = M; R.first = first; R.n = n; R.Rcap = e->Rcap;
    const int grid = e->n_sm;
    const int nw = grid * (RW_THREADS / 32);
    // events per member below a step's frontier: about three tests per warp and step, never more than half a window
    R.L = std::max(1, std::min(RW_LMAX / 2, 3 * nw * e->nranks / std::max(1, M)));
    R.epoch = ++e->rb_epoch;
    R.row = e->d_row.get(); R.p0 = e->d_p0.get(); R.creator = e->d_creator.get(); R.seq = e->d_seq.get(); R.round = e->d_round.get();
    R.Wf = e->d_Wf.get(); R.scw = e->d_scw.get(); R.sctag = e->d_sctag.get(); R.cev = T.cev;
    R.cmin = T.cmin; R.coff = T.coff; R.bar = T.bar; R.ticket = rb_meta(e->d_rbmeta.get(), e->MP).ticket;
    R.ctot = T.ctot; R.gchain = T.gchain; R.hitmin = e->d_hitmin.get();
    R.stake = e->d_stake.get(); R.tot2 = 2 * e->tot; R.unit = e->unit ? 1 : 0; R.scal = e->d_scal.get(); R.dbg = e->d_dbg.get();
    R.rank = e->rank; R.nranks = e->nranks; R.xstep = e->d_xstep.get();
    for (int p = 0; p < e->nranks && p < 8; p++) {
        R.xflag[p] = reinterpret_cast<unsigned *>(e->x_peer[p]);
        R.xhit[p] = reinterpret_cast<u64 *>(reinterpret_cast<char *>(e->x_peer[p]) + 256);
    }
    const size_t smem = rounds_wide_smem(M);
    CK(cudaFuncSetAttribute(k_rounds_wide<NJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    void *args[] = {(void *)&R};
    {
        Span sp(e, e->stream.get(), SpanCat::rounds);
        CK(cudaLaunchCooperativeKernel((void *)k_rounds_wide<NJ>, dim3(grid), dim3(RW_THREADS), args, smem, e->stream.get()));
    }
    k_rb_finish<<<std::max(1, std::min(2 * e->n_sm, (n + 255) / 256)), 256, 0, e->stream.get()>>>(T, RbFold{});
    k_w_seenmask<NJ><<<std::max(1, std::min(8 * e->n_sm, (n + 7) / 8)), 256, 0, e->stream.get()>>>(M, first, n, e->Rcap, e->d_row.get(), e->d_round.get(), e->d_W.get(), e->d_SMw.get());
    CK(cudaGetLastError());
    StrongParams Q{};
    Q.M = M; Q.first = first; Q.n = n; Q.Rcap = e->Rcap; Q.creator = e->d_creator.get(); Q.row = e->d_row.get();
    Q.round = e->d_round.get(); Q.wit = e->d_wit.get(); Q.stake = e->d_stake.get(); Q.tot2 = 2 * e->tot;
    Q.coin = e->d_coin.get(); Q.sig = e->d_sig.get(); Q.unit = e->unit ? 1 : 0; Q.list = T.wlist; Q.list_n = T.wcnt;
    Q.SMw = e->d_SMw.get(); Q.Sw = e->d_Sw.get();
    const size_t ssm = (size_t)(2 * M + 8 * M) * sizeof(int);
    CK(cudaFuncSetAttribute(k_w_strong<NJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssm));
    k_w_strong<NJ><<<std::max(1, std::min(4 * e->n_sm, (n + 7) / 8)), 256, ssm, e->stream.get()>>>(Q);
    CK(cudaGetLastError());
    e->stats.kernel_launches += 4;
    return 0;
}

size_t w_fame_smem(int NJ, int M) { return (size_t)(32 * NJ + 64) * sizeof(int) + (size_t)(32 + M) * sizeof(i64); }

template <int NJ, class Src>
int fame_rounds_wide(sw_engine *e, Src P, int B) {
    const int parts = (e->M + FW_THREADS - 1) / FW_THREADS;
    k_w_fame_rounds<NJ><<<dim3((2 * e->n_sm / parts + 1) * parts, B), FW_THREADS, w_fame_smem(NJ, e->M), e->stream.get()>>>(P);
    return 0;
}

// The fame kernels of B views: P is one view's parameters (B = 1) or the device array of B views' (swirld_kernels.cuh,
// params).  Every view gets the grid its single call launches (the kernels are latency-bound; spare CTAs exit at once).
template <class Src>
void fame_kernels(sw_engine *e, Src P, int B) {
    if (e->wide) {
        k_fame_begin<<<dim3(1, B), 32, 0, e->stream.get()>>>(P);
        SW_NJ(fame_rounds_wide, e, P, B);
        k_fame_finish<<<dim3(1, B), 1024, 0, e->stream.get()>>>(P);
        e->stats.kernel_launches += 3;
    } else {
        k_fame_rounds<<<dim3(2 * e->n_sm, B), 256, 0, e->stream.get()>>>(P);
        e->stats.kernel_launches += 1;
    }
}

// decide_fame copies the scalars and (speculatively) the first new consensus rounds together: one copy, one
// synchronisation (a 64-member chunk of 64 K events brings about 90 new rounds: room for 64 only would add a copy and a
// synchronisation to every such call)
constexpr int FAME_SPEC = 1024;
int fame_spec(const sw_engine *e) { return std::min(e->Rcap, FAME_SPEC); }

// find_order's output comes back the same way: the first events a call orders, with their consensus times and rounds
// received (OrderOut, 4 ints each), wait behind the scalars in the room of the new rounds (decide_fame has copied
// those back before any find_order runs) and ride on the copy of the scalars.  The window is what the call can order at
// most, n_divided - n_transactions, up to ORDER_SPEC; a call that orders more copies the rest from the columns.
constexpr int ORDER_SPEC = 1024;
int order_spec(const sw_engine *e) { return std::min(e->n_divided - e->n_tx, ORDER_SPEC); }
size_t scal_room(const sw_engine *e) { return (size_t)std::max(e->Rcap, 4 * ORDER_SPEC); }   // ints behind the scalars

// What decide_fame does once that copy is in h_scal: `r` = the error the device found, or the count of new rounds,
// which go to `out` (a second copy when more came than the first one held).  Returns < 0 only when a copy fails.
int fame_result(sw_engine *e, int32_t *out, int cap, int &r) {
    r = device_error(e);
    if (r < 0) return 0;
    const int cnt = e->h_scal.get()[SC_NEWC];
    if (cnt > cap) { r = fail(e, SW_E_ARG, "decide_fame: %d new consensus rounds do not fit cap=%d", cnt, cap); return 0; }
    if (cnt > fame_spec(e)) {
        CK(cudaMemcpyAsync(e->h_newc, e->d_newc, sizeof(int32_t) * cnt, cudaMemcpyDeviceToHost, e->stream.get()));
        CK(cudaStreamSynchronize(e->stream.get()));
        e->stats.d2h_bytes += sizeof(int32_t) * cnt;
    }
    if (cnt > 0) memcpy(out, e->h_newc, sizeof(int32_t) * cnt);
    r = cnt;
    return 0;
}

FameParams fame_params(const sw_engine *e) {
    FameParams P{};
    P.M = e->M; P.Rcap = e->Rcap; P.C = e->C; P.W = e->d_W.get(); P.S = e->d_S.get(); P.famous = e->d_famous.get();
    P.famous_ev = e->d_famous_ev.get(); P.consensus = e->d_consensus.get(); P.done = e->d_done.get(); P.rem = e->d_rem.get();
    P.coin = e->d_coin.get(); P.stake = e->d_stake.get(); P.tot2 = 2 * e->tot; P.unit = e->unit ? 1 : 0; P.newc = e->d_newc; P.scal = e->d_scal.get();
    P.Sw = e->d_Sw.get();
    return P;
}

// find_order's per-round scratch, grown on demand to n rounds
size_t seg_cap(const sw_engine *e) { return e->d_seg_nf.cap(); }
int order_scratch(sw_engine *e, int n) {
    const size_t nc = std::max<size_t>(n, std::max<size_t>(64, 2 * seg_cap(e))), MS = e->MS;
    return grow(e, n, seg_cap(e), sized(e->d_seg_start, nc + 1), sized(e->d_seg_fw, nc * MS), sized(e->d_seg_nf, nc),
                sized(e->d_seg_white, nc * 64), sized(e->d_rounds_in, nc), sized(e->d_plan, nc * MS * 8));
}

// find_order over the n sorted rounds at `rounds` (device memory)
OrderParams order_params(const sw_engine *e, int n, const int32_t *rounds) {
    OrderParams P{};
    P.M = e->M; P.Rcap = e->Rcap; P.nrounds = n; P.rounds = rounds; P.W = e->d_W.get(); P.famous = e->d_famous.get();
    P.row = e->d_row.get(); P.p0 = e->d_p0.get(); P.creator = e->d_creator.get(); P.seq = e->d_seq.get(); P.t = e->d_t.get(); P.sig = e->d_sig.get();
    P.stake = e->d_stake.get(); P.tot = e->tot; P.lastord = e->d_lastord.get(); P.batch_ev = e->d_batch_ev.get(); P.batch_seg = e->d_batch_seg.get();
    P.seg_start = e->d_seg_start.get(); P.seg_fw = e->d_seg_fw.get(); P.seg_nf = e->d_seg_nf.get(); P.seg_white = e->d_seg_white.get();
    P.ts = e->d_ts.get(); P.key = e->d_key.get(); P.perm = e->d_perm.get(); P.tx = e->d_tx.get(); P.tx_cap = e->cap;
    P.idx = e->d_idx.get(); P.tx_base = e->n_tx; P.scal = e->d_scal.get(); P.out_n = 0;
    P.plan = e->d_plan.get(); P.plan_stride = (int)(seg_cap(e) * e->MS);
    return P;
}

// sorted(new_c) (swirld.py:283) of n rounds, in place; false when one is not in the round table (`bad`: the first)
bool sort_rounds(const sw_engine *e, int32_t *rs, int n, int &bad) {
    std::sort(rs, rs + n);
    for (int i = 0; i < n; i++)
        if (rs[i] < 0 || rs[i] >= e->Rcap) { bad = rs[i]; return false; }
    return true;
}

// The five order kernels of A views (P: as fame_kernels), every view's grid sized from `maxn` rounds.  The number of
// newly ordered events stays on the device: the time and sort kernels read it there, the host learns it from the
// copy at the end of the call.
template <class Src>
void order_kernels(sw_engine *e, Src P, int A, int maxn) {
    const int M = e->M;
    const int list_ctas = std::max(1, std::min(4 * e->n_sm, (int)(((size_t)maxn * e->MS + 255) / 256)));
    if (e->wide) {
        k_w_order_rounds<<<dim3(maxn, A), 1024, (size_t)3 * M * sizeof(int), e->stream.get()>>>(P);
        k_w_order_cuts<<<dim3(1, A), 1024, (size_t)2 * M * sizeof(int), e->stream.get()>>>(P);
        k_w_order_list<<<dim3(list_ctas, A), 256, 0, e->stream.get()>>>(P);
        k_w_order_times<<<dim3(8 * e->n_sm, A), OW_WARPS * 32, (size_t)OW_WARPS * M * sizeof(u64), e->stream.get()>>>(P);
    } else {
        k_order_rounds<<<dim3(maxn, A), 1024, 0, e->stream.get()>>>(P);
        k_order_cuts<<<dim3(1, A), 64, 0, e->stream.get()>>>(P);
        k_order_list<<<dim3(list_ctas, A), 256, 0, e->stream.get()>>>(P);
        k_order_times<<<dim3(4 * e->n_sm, A), 256, 0, e->stream.get()>>>(P);
    }
    k_order_sort<<<dim3(maxn, A), 1024, 0, e->stream.get()>>>(P);
    e->stats.kernel_launches += 5;
}

// what find_order does once its copy of the scalars is in h_scal: the error the device found, else the events it ordered
int order_result(sw_engine *e) {
    const int rc = device_error(e);
    if (rc < 0) return rc;
    const int nbatch = e->h_scal.get()[SC_BATCH];
    e->n_tx += nbatch;
    return nbatch;
}

// The output of a find_order call that ordered the positions [base, base + cnt), of which the first `staged` came back
// in `st`, into ev/ts/rr[0, cnt): the rest is copied from the columns on stream `s` (the caller synchronises it once).
int order_output(sw_engine *e, cudaStream_t s, int base, int cnt, const OrderOut *st, int staged,
                 int32_t *ev, double *ts, int32_t *rr) {
    const int k = std::min(cnt, staged);
    for (int i = 0; i < k; i++) { ev[i] = st[i].ev; ts[i] = st[i].ts; rr[i] = st[i].rr; }
    if (cnt > k) {
        const size_t n = cnt - k, at = (size_t)base + k;
        CK(cudaMemcpyAsync(ev + k, e->d_tx.get() + at, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(ts + k, e->d_tx_ts + at, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(rr + k, e->d_tx_rr + at, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, s));
    }
    return cnt - k;
}

// ---- several node-views per call (sw_batch_*)
// The checks shared by the batched calls: they refuse the whole batch before anything runs (the message goes to the first
// engine).  `same_shape`: the views must also share M and the kernel family (all but sw_batch_append).
// `drain`: give up the views' round-stream pieces (every call that writes consensus state; the sync calls only read rows)
int check_views(sw_engine *const *engines, int B, const char *what, bool same_shape, bool drain = true) {
    sw_engine *e = engines[0];
    std::vector<const sw_engine *> seen(engines, engines + B);
    for (int v = 0; v < B; v++)
        if (!engines[v]) return fail(e, SW_E_ARG, "%s: view %d is NULL", what, v);
    std::sort(seen.begin(), seen.end());
    if (std::adjacent_find(seen.begin(), seen.end()) != seen.end()) return fail(e, SW_E_ARG, "%s: an engine appears twice", what);
    for (int v = 0; v < B; v++) {
        const sw_engine *x = engines[v];
        if (x->device != e->device || (same_shape && (x->M != e->M || x->wide != e->wide)))
            return fail(e, SW_E_UNSUPPORTED, "%s: view %d: the views must %s on one device", what, v,
                        same_shape ? "have one member count and one kernel family" : "be");
        if (x->nranks > 1) return fail(e, SW_E_UNSUPPORTED, "%s: view %d is one rank of a multi-GPU engine", what, v);
    }
    for (int v = 0; v < B && drain; v++)
        if (rs_drain(engines[v]) < 0) { e->err = engines[v]->err; return SW_E_CUDA; }
    return 0;
}

// the per-call block of the first engine: at least `bytes` on the device and in pinned host memory
int views_buffer(sw_engine *e, size_t bytes) {
    const size_t want = std::max(bytes, 2 * e->d_vbuf.cap());
    return grow(e, bytes, e->d_vbuf.cap(), sized(e->d_vbuf, want), sized(e->h_vbuf, want));
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// The next slot of at least `bytes` in the staging ring, once the copy that used it STAGE_SLOTS calls ago is done (a
// larger ring replaces the ring after the copies and kernels that read it).  Returns the slot's index (< 0: an error);
// the caller records stage_ev[slot] on the copy stream after its copy.
int stage_slot(sw_engine *e, size_t bytes) {
    const size_t ring = align256(std::max(bytes, 2 * e->stage_bytes())) * sw_engine::STAGE_SLOTS;
    if (grow(e, bytes, e->stage_bytes(), sized(e->h_stage, ring), sized(e->d_stage, ring)) < 0) return SW_E_CUDA;
    const int si = e->stage_next;
    e->stage_next = (si + 1) % sw_engine::STAGE_SLOTS;
    CK(cudaEventSynchronize(e->stage_ev[si].get()));
    return si;
}

// the batch runs on the stream of `e`, the first engine: after everything each view has queued on its own
int views_enter(sw_engine *e, sw_engine *const *views, int B) {
    for (int v = 0; v < B; v++)
        if (views[v] != e && follow(views[v], views[v]->stream.get(), e->stream.get()) < 0) { e->err = views[v]->err; return SW_E_CUDA; }
    return 0;
}

// ... and each view's next call runs after what the batch has queued there so far
int views_resume(sw_engine *e, sw_engine *const *views, int B) {
    std::vector<cudaStream_t> others;
    for (int v = 0; v < B; v++) if (views[v] != e) others.push_back(views[v]->stream.get());
    return follow(e, e->stream.get(), others, e->view_ev.get());
}

// the views resume; then the one copy of the gathered scalars and the one synchronisation
int views_leave(sw_engine *e, sw_engine *const *views, int B, void *h_dst, const void *d_src, size_t bytes) {
    if (views_resume(e, views, B) < 0) return SW_E_CUDA;
    CK(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, e->stream.get()));
    CK(cudaStreamSynchronize(e->stream.get()));
    e->stats.d2h_bytes += bytes;
    return 0;
}

// sw_create and sw_load: `wide` selects the any-M kernels (swirld_wide.cuh), required above 64 members.  Nothing here
// changes state that other engines of the process share.
int create(int M, int capacity_events, const int64_t *stake, int coin_period, int device, bool wide, sw_engine **out) {
    sw_engine *e = nullptr;
    if (!out) return fail(e, SW_E_ARG, "out is NULL");
    *out = nullptr;
    if (M < 1 || capacity_events < 1 || coin_period < 1) return fail(e, SW_E_ARG, "bad M / capacity / coin period");
    if (M > SW_MAX_MEMBERS) return fail(e, SW_E_UNSUPPORTED, "M=%d > %d members not supported by this build", M, SW_MAX_MEMBERS);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1)
        return fail(e, SW_E_CUDA, "no CUDA device (this engine has no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(e, SW_E_ARG, "device %d out of range (%d devices)", device, ndev);
    e = new sw_engine();
    e->M = M; e->NC = (M + 31) / 32; e->cap = capacity_events; e->C = coin_period; e->device = device;
    e->wide = wide;
    e->NJ = 1;
    while (e->NJ * 32 < M) e->NJ *= 2;
    e->MS = e->wide ? M : 64;
    e->MP = std::max(M, 64);
    e->h_stake.resize(M);
    for (int c = 0; c < M; c++) {
        e->h_stake[c] = stake ? stake[c] : 1;
        if (e->h_stake[c] < 0) { delete e; return fail(nullptr, SW_E_ARG, "negative stake"); }
        if (e->h_stake[c] != 1) e->unit = false;
        // the fame and round tests compare 3 * (a sum of stakes) with 2 * tot in int64: refuse totals whose triple overflows
        if (__builtin_add_overflow(e->tot, e->h_stake[c], &e->tot) || e->tot > INT64_MAX / 3) {
            delete e; return fail(nullptr, SW_E_ARG, "total stake above (2^63 - 1) / 3");
        }
    }
    // a round other than the last needs more than 2*tot/3 members with a witness (quirk Q3)
    i64 per = std::min<i64>(M, (2 * e->tot) / 3 + 1);
    if (per < 1) per = 1;
    e->Rcap = (int)std::min<i64>((i64)e->cap + 2, (i64)e->cap / per + 16);
    e->h_head.assign(M, -1);
    e->h_count.assign(M, 0);
    e->h_creator.reserve(e->cap);
    e->h_stale_cum.assign(1, 0);
    int rc = [&]() -> int {
        CK(cudaSetDevice(device));
        CK(e->stream.create()); CK(e->copy_stream.create());
        CK(e->scan_ev.create()); CK(e->view_ev.create());
        for (Event &ev : e->stage_ev) CK(ev.create());
        const size_t cap = e->cap, RM = (size_t)e->Rcap * M, MP = e->MP;
        CK(e->h_height.alloc(cap)); CK(e->h_seq.alloc(cap)); CK(e->h_stale.alloc(cap));
        CK(e->d_p0.alloc(cap)); CK(e->d_p1.alloc(cap)); CK(e->d_creator.alloc(cap)); CK(e->d_seq.alloc(cap));
        CK(e->d_t.alloc(cap)); CK(e->d_sig.alloc(cap * 64)); CK(e->d_height.alloc(cap)); CK(e->d_stale.alloc(cap));
        // can_see scan scratch: per-event meta / flags / slow list, per-block tables (blocks are >= cs_min_B events)
        e->cs_min_B = std::max(256, std::min((M <= 64 ? 16 : 32) * M, 1 << 15));
        const size_t nbmax = cap / e->cs_min_B + 3;
        CK(e->d_cs_meta.alloc(cap)); CK(e->d_cs_wr.alloc(cap)); CK(e->d_cs_xb.alloc(cap)); CK(e->d_cs_slow.alloc(cap + 4));
        CK(e->d_cs_last.alloc(nbmax * M)); CK(e->d_cs_Q.alloc((nbmax + 1) * M)); CK(e->d_cs_slowcnt.alloc(4)); CK(e->d_cs_sflag.alloc(cap)); CK(e->d_cs_xlist.alloc(cap + 4)); CK(e->d_cs_slowblk.alloc(cap + 4)); CK(e->d_cs_blkcnt.alloc(nbmax + 1));
        CK(e->d_cs_carry.alloc(MP));
        CK(e->d_Wf.alloc(RM)); CK(e->d_cev.alloc(2 * cap)); /* + the witness list of the current chunk */
        CK(e->d_rbmeta.alloc(rb_meta_ints(e->MP)));
        CK(e->d_rbtot.alloc(MP)); CK(e->d_gchain.alloc(MP * RB_RING));
        CK(cudaDeviceGetAttribute(&e->n_sm, cudaDevAttrMultiProcessorCount, device));
        CK(e->d_dbg.alloc(40)); CK(cudaMemsetAsync(e->d_dbg.get(), 0, sizeof(long long) * 40, e->stream.get()));
        CK(e->d_row.alloc(cap * M));
        if (e->wide) {
            CK(e->d_scw.alloc(cap * e->NJ)); CK(e->d_sctag.alloc(cap)); CK(e->d_SMw.alloc(cap * e->NJ));
            CK(e->d_Sw.alloc(RM * e->NJ)); CK(e->d_hitmin.alloc((size_t)3 * M));
            CK(e->d_xbuf.alloc(256 + (size_t)8 * 3 * M * sizeof(u64)));
            CK(cudaMemsetAsync(e->d_xbuf.get(), 0, 256 + (size_t)8 * 3 * M * sizeof(u64), e->stream.get()));
            CK(e->d_xstep.alloc(1)); CK(cudaMemsetAsync(e->d_xstep.get(), 0, sizeof(unsigned), e->stream.get()));
            e->x_peer[0] = e->d_xbuf.get();
        } else {
            CK(e->d_sc.alloc(cap)); CK(e->d_res.alloc((size_t)2 * 64 * RB_LMAX));
            CK(e->d_SM.alloc(cap)); CK(e->d_S.alloc(RM));
            // the cluster round kernel: 16 CTAs with ~174 KB of shared memory each must fit one GPC
            CK(e->d_rccont.alloc(132)); CK(cudaMemsetAsync(e->d_rccont.get(), 0, sizeof(int32_t) * 132, e->stream.get()));
            bool want = true;
            if (const char *v = getenv("SW_ROUNDS_CLUSTER")) want = atoi(v) != 0;
            if (const char *v = getenv("SW_RC_MIN_N")) e->rc_min_n = std::max(1, atoi(v));
            if (const char *v = getenv("SW_RC_STEPS")) {         // profiling: log this many cluster steps per CTA
                const unsigned cap = (unsigned)std::max(0, atoi(v));
                const size_t words = RC_LOGH + (size_t)cap * RC_CS * RC_NLOG;
                CK(e->d_rcslog.alloc(words)); CK(cudaMemsetAsync(e->d_rcslog.get(), 0, sizeof(unsigned) * words, e->stream.get()));
                CK(cudaMemcpyAsync(e->d_rcslog.get() + 1, &cap, sizeof(unsigned), cudaMemcpyHostToDevice, e->stream.get()));
                CK(cudaStreamSynchronize(e->stream.get()));
            }
            if (want) {
                int ncl = 0;
                const cudaError_t er = SW_NCU(e, rc_setup, &ncl);
                e->rc_ok = er == cudaSuccess && ncl >= 1;
                if (er != cudaSuccess) (void)cudaGetLastError();
            }
            bool ahead = e->rc_ok;
            if (const char *v = getenv("SW_ROUNDS_AHEAD")) ahead = ahead && atoi(v) != 0;
            if (ahead && rs_create(e) < 0) return SW_E_CUDA;
        }
        CK(e->d_round.alloc(cap)); CK(e->d_wit.alloc(cap)); CK(e->d_famous_ev.alloc(cap));
        CK(e->d_W.alloc(RM)); CK(e->d_famous.alloc(RM));
        CK(e->d_consensus.alloc(e->Rcap)); CK(e->d_done.alloc(e->Rcap)); CK(e->d_coin.alloc(RM));
        CK(e->d_rem.alloc(e->Rcap));
        CK(e->d_stake.alloc(M)); CK(e->d_scal.alloc(SC_COUNT + scal_room(e)));
        e->d_newc = e->d_scal.get() + SC_COUNT;                  // (sw_decide_fame copies the scalars and the new rounds at once)
        CK(e->d_lastord.alloc(MP)); CK(e->d_tx.alloc(4 * cap)); CK(e->d_idx.alloc(cap));
        e->d_tx_rr = e->d_tx.get() + cap;                        // (one block: OrderParams finds both from d_tx and cap)
        e->d_tx_ts = reinterpret_cast<double *>(e->d_tx.get() + 2 * cap);
        CK(e->d_batch_ev.alloc(cap)); CK(e->d_batch_seg.alloc(cap)); CK(e->d_perm.alloc(2 * cap));
        CK(e->d_ts.alloc(cap)); CK(e->d_key.alloc(cap * 8));
        if (stage_slot(e, unpack_bytes(sw_engine::STAGE_EVENTS)) < 0) return SW_E_CUDA;   // (the ring, sized for sw_append)
        CK(cudaFuncSetAttribute(k_stream_divide<true, StreamParams>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 1024));
        CK(cudaFuncSetAttribute(k_stream_divide<true, const StreamParams *>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 1024));
        CK(e->h_scal.alloc(SC_COUNT + scal_room(e)));
        e->h_newc = e->h_scal.get() + SC_COUNT;
        CK(cudaMemcpyAsync(e->d_stake.get(), e->h_stake.data(), sizeof(i64) * M, cudaMemcpyHostToDevice, e->stream.get()));
        // kernels that need more than the default 48 KB of dynamic shared memory: the limit is a property of the kernel in
        // the whole process, so it is what the largest member count needs, whatever M this engine has
        const size_t cs_smem = (size_t)(SW_MAX_MEMBERS + CS_SV) * CS_CT * sizeof(int) + CS_TILE * sizeof(int4) + 3 * CS_TILE;
        CK(cudaFuncSetAttribute(k_cs_pass<1, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_pass<2, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_pass<1, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_pass<2, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_pass<1, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_pass<2, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_pass<1, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_pass<2, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cs_smem));
        CK(cudaFuncSetAttribute(k_cs_slow_wave, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)CS_SLOW_WARPS * SW_MAX_MEMBERS * sizeof(int))));
        CK(cudaFuncSetAttribute(k_cs_slow_rest, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)CS_REST_WARPS * SW_MAX_MEMBERS * sizeof(int))));
        return reset_state(e);
    }();
    if (rc < 0) { g_create_error = e->err; sw_destroy(e); return rc; }
    memset(&e->stats, 0, sizeof e->stats);
    *out = e;
    return SW_OK;
}

// ---- the parts of sw_append, shared with sw_batch_append
// The graph-shape checks of is_valid_event (swirld.py:104-108) and the fork-free contract for the n events that follow
// the engine's last one, updating the host mirrors; on an error the mirrors are as they were and the message is the
// engine's.
int append_validate(sw_engine *e, int n, const int32_t *p0, const int32_t *p1, const int32_t *creator) {
    if ((i64)e->n_events + n > e->cap) return fail(e, SW_E_CAPACITY, "capacity_events=%d exceeded", e->cap);
    const int base = e->n_events;
    std::vector<int32_t> head_save(e->h_head), count_save(e->h_count);
    e->h_creator.resize((size_t)base + n);
    int rc = SW_OK;
    int next_snap = (base / sw_engine::SNAP + 1) * sw_engine::SNAP;
    for (int j = 0; j < n && rc == SW_OK; j++) {
        const int i = base + j, c = creator[j], a = p0[j], b = p1[j];
        if (c < 0 || c >= e->M) { rc = fail(e, SW_E_ARG, "event %d: creator %d out of range", i, c); break; }
        e->h_stale.get()[i] = 0;
        if (a < 0 && b < 0) {
            if (e->h_head[c] >= 0) { rc = fail(e, SW_E_FORK, "event %d: second root of member %d", i, c); break; }
            e->h_height.get()[i] = 0;                                          // swirld.py:117-118
        } else {
            if (a < 0 || b < 0 || a >= i || b >= i) { rc = fail(e, SW_E_PARENT, "event %d: parents (%d,%d) unknown", i, a, b); break; }
            if (e->h_creator[a] != c) { rc = fail(e, SW_E_PARENT, "event %d: self-parent %d has another creator", i, a); break; }
            if (e->h_creator[b] == c) { rc = fail(e, SW_E_PARENT, "event %d: other-parent %d has the same creator", i, b); break; }
            if (e->h_head[c] != a) { rc = fail(e, SW_E_FORK, "event %d: self-parent %d is not member %d's latest event (fork)", i, a, c); break; }
            e->h_height.get()[i] = std::max(e->h_height.get()[a], e->h_height.get()[b]) + 1;   // swirld.py:120
            e->h_stale.get()[i] = e->h_head[e->h_creator[b]] != b;             // "near fork": an older event of the peer
        }
        e->h_creator[i] = c;
        e->h_head[c] = i;
        e->h_seq.get()[i] = e->h_count[c]++;
        if (i + 1 == next_snap) { push_snapshot(e, i + 1, e->h_count); next_snap += sw_engine::SNAP; }
    }
    if (rc != SW_OK) {
        e->h_head = head_save; e->h_count = count_save;
        e->h_creator.resize(base);
        while (!e->snap_at.empty() && e->snap_at.back() > base) { e->snap_at.pop_back(); e->snap_cnt.resize(e->snap_at.size() * e->M); }
        return rc;
    }
    e->h_stale_cum.resize((size_t)base + n + 1);
    for (int j = 0; j < n; j++) e->h_stale_cum[base + j + 1] = e->h_stale_cum[base + j] + e->h_stale.get()[base + j];
    return SW_OK;
}

// A handful of events (at most STAGE_EVENTS): the eight columns packed at `hs` (unpack_bytes(n) bytes, which go to
// `ds` on the device), and what k_unpack needs to scatter them.  The caller's arrays are free once this returns.
UnpackParams append_pack(const sw_engine *e, int n, const int32_t *p0, const int32_t *p1, const int32_t *creator,
                         const double *t, const uint8_t *sig, uint8_t *hs, const uint8_t *ds) {
    const int base = e->n_events;
    int32_t *ints = reinterpret_cast<int32_t *>(hs);
    memcpy(ints, p0, sizeof(int32_t) * n); memcpy(ints + n, p1, sizeof(int32_t) * n); memcpy(ints + 2 * n, creator, sizeof(int32_t) * n);
    memcpy(ints + 3 * n, e->h_seq.get() + base, sizeof(int32_t) * n); memcpy(ints + 4 * n, e->h_height.get() + base, sizeof(int32_t) * n);
    uint8_t *pt = hs + unpack_off_t(n);
    memcpy(pt, t, sizeof(double) * n); memcpy(pt + (size_t)8 * n, sig, (size_t)64 * n); memcpy(pt + (size_t)72 * n, e->h_stale.get() + base, (size_t)n);
    UnpackParams U{};
    U.base = base; U.n = n; U.stage = ds; U.p0 = e->d_p0.get(); U.p1 = e->d_p1.get(); U.creator = e->d_creator.get(); U.seq = e->d_seq.get();
    U.height = e->d_height.get(); U.t = e->d_t.get(); U.sig = e->d_sig.get(); U.stale = e->d_stale.get();
    return U;
}

// The first `bytes` of slot `si` of the staging ring go over on the copy stream and one k_unpack scatters them: U is one
// view's parameters (B = 1) or the device array of B views' at the start of the slot
template <class Src>
int unpack_staged(sw_engine *e, int si, size_t bytes, Src U, int B) {
    cudaStream_t cs = e->copy_stream.get();
    CK(cudaMemcpyAsync(e->d_stage.get() + e->stage_bytes() * si, e->h_stage.get() + e->stage_bytes() * si, bytes, cudaMemcpyHostToDevice, cs));
    CK(cudaEventRecord(e->stage_ev[si].get(), cs));
    k_unpack<<<dim3(1, B), 256, 0, cs>>>(U);
    CK(cudaGetLastError());
    e->stats.kernel_launches += 1;
    return 0;
}

// More events: one copy per column on the engine's copy stream (from pinned memory, asynchronous)
int append_copy(sw_engine *e, int n, const int32_t *p0, const int32_t *p1, const int32_t *creator, const double *t,
                const uint8_t *sig) {
    const int base = e->n_events;
    cudaStream_t cs = e->copy_stream.get();
    CK(cudaMemcpyAsync(e->d_p0.get() + base, p0, sizeof(int32_t) * n, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(e->d_p1.get() + base, p1, sizeof(int32_t) * n, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(e->d_creator.get() + base, creator, sizeof(int32_t) * n, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(e->d_t.get() + base, t, sizeof(double) * n, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(e->d_sig.get() + (size_t)base * 64, sig, (size_t)64 * n, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(e->d_seq.get() + base, e->h_seq.get() + base, sizeof(int32_t) * n, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(e->d_height.get() + base, e->h_height.get() + base, sizeof(int32_t) * n, cudaMemcpyHostToDevice, cs));
    CK(cudaMemcpyAsync(e->d_stale.get() + base, e->h_stale.get() + base, (size_t)n, cudaMemcpyHostToDevice, cs));
    return 0;
}

// The n validated events are queued on `st` (the engine's copy stream, or the first engine's for a packed batch): count
// them, and start their can_see rows when the batch is big.  Later calls wait for `st` at this point (wait_appends).
int append_commit(sw_engine *e, int n, cudaStream_t st) {
    const int base = e->n_events;
    // rows are up to date and the batch is big: scan it now, beside the kernels of the previous chunk
    // (several ranks: the scan holds cross-GPU barriers; it must not run beside a round kernel that fills every SM while
    //  waiting for the same peer -- scans stay on the compute stream then)
    const bool eager = e->n_rowed == base && n >= 4096 && e->nranks == 1;
    e->stats.h2d_bytes += (i64)n * (5 * 4 + 1 + 8 + 64);
    e->stats.events += n;
    e->n_events += n;
    push_append_snapshot(e);
    if (eager) {
        if (e->scan_ev_set) CK(cudaStreamWaitEvent(st, e->scan_ev.get(), 0));     // never beside a scan on the compute stream
        int rc2 = cansee_scan(e, st, e->n_events);
        if (rc2 < 0) return rc2;
    }
    // the compute stream waits for this batch only when a call first touches it (wait_appends)
    Event done = get_event(e);
    CK(cudaEventRecord(done.get(), st));
    e->appends.push_back({base, std::move(done)});
    return 0;
}

// divide_rounds of [first, first+n) in one launch of k_stream_divide (swirld_stream.cuh)
StreamParams stream_params(const sw_engine *e, int first, int n) {
    StreamParams S{};
    S.M = e->M; S.first = first; S.n = n; S.Rcap = e->Rcap; S.NJ = e->NJ;
    S.p0 = e->d_p0.get(); S.p1 = e->d_p1.get(); S.creator = e->d_creator.get(); S.seq = e->d_seq.get(); S.row = e->d_row.get(); S.round = e->d_round.get();
    S.wit = e->d_wit.get(); S.W = e->d_W.get(); S.Wf = e->d_Wf.get(); S.SM = e->d_SM.get(); S.S = e->d_S.get(); S.SMw = e->d_SMw.get(); S.Sw = e->d_Sw.get();
    S.coin = e->d_coin.get(); S.sig = e->d_sig.get(); S.stake = e->d_stake.get(); S.tot2 = 2 * e->tot; S.scal = e->d_scal.get();
    S.ctot = e->d_rbtot.get(); S.gchain = e->d_gchain.get(); S.carry = e->d_cs_carry.get(); S.ring = RB_RING;
    return S;
}
int stream_threads(int M) { return std::min(1024, std::max(32, (M + 31) / 32 * 32)); }
size_t stream_smem(int M) { return (size_t)M * 8 + 32 * 8 + (size_t)3 * M * 4 + 32 * 4; }

// The one launch: S is one view's parameters (B = 1) or the device array of B views' (swirld_kernels.cuh, params)
template <class Src>
int stream_kernel(sw_engine *e, Src S, int B) {
    {
        Span sp(e, e->stream.get(), SpanCat::divide);
        if (e->wide) k_stream_divide<true><<<dim3(1, B), stream_threads(e->M), stream_smem(e->M), e->stream.get()>>>(S);
        else k_stream_divide<false><<<dim3(1, B), stream_threads(e->M), stream_smem(e->M), e->stream.get()>>>(S);
        CK(cudaGetLastError());
    }
    e->stats.kernel_launches += 1;
    return 0;
}

// the reference's own cadence (one sync per call): a call of at most STREAM_N events whose rows are current is divided
// in ONE launch (swirld_stream.cuh)
bool stream_path(const sw_engine *e, int first, int n) { return n <= sw_engine::STREAM_N && e->n_rowed == first; }

// Before a chunk [first, first+n) on the compute stream: rows behind (small appends, or after sw_rewind) are scanned
// there, for everything appended so far and after the copies of EVERY appended batch (the scan reads the columns of
// all of them); else the stream waits for the copies of the batches the chunk touches.
// `upto` < n_events: scan only so far (the ahead path scans the rest beside the call's piece).
int rows_ready(sw_engine *e, int first, int n, int upto = -1) {
    if (first + n <= e->n_rowed) return wait_appends(e, first + n);
    if (wait_appends(e, -1) < 0) return SW_E_CUDA;
    const int rc = cansee_scan(e, e->stream.get(), upto < 0 ? e->n_events : upto);
    return rc < 0 ? rc : rows_written(e);
}

void divided(sw_engine *e, int n) {
    e->stats.events_divided += n;
    e->n_divided += n;
}

// what a call on the streaming path leaves behind: its rows are complete (written on the compute stream)
int stream_divided(sw_engine *e, int n) {
    e->n_rowed = e->n_divided + n;
    if (rows_written(e) < 0) return SW_E_CUDA;
    divided(e, n);
    return 0;
}

// The chunk path of sw_batch_divide_rounds (M <= 64, one stake shape): every step of a view runs on the view's own
// stream, except the round kernels, which advance side by side in ONE cooperative launch on the stream of `e`, the
// first engine of the batch (its parameter buffers; it is charged the timings and launches).
template <int NC, bool UNIT>
int chunk_views(sw_engine *e, sw_engine *const *engines, int B, const int *first, const int *n) {
    const int per_launch = e->n_sm;                         // (one CTA per view at least: its warps loop over its chains)
    if (grow(e, B, e->d_views.cap(), sized(e->d_views, B), sized(e->d_rcviews, B)) < 0) return SW_E_CUDA;
    // one thread-block cluster per view first (swirld_rcluster.cuh); the grid-wide kernel then takes what they hand back
    bool use_rc = true;
    for (int v = 0; v < B; v++) use_rc = use_rc && engines[v]->rc_ok && n[v] >= e->rc_min_n;
    std::vector<RcParams> Qv(B);
    std::vector<RbParams> Rv(B);
    for (int v0 = 0; v0 < B; v0 += per_launch) {
        const int nv = std::min(per_launch, B - v0), G = e->n_sm / nv;
        for (int v = v0; v < v0 + nv; v++) {
            sw_engine *x = engines[v];
            if (rows_ready(x, first[v], n[v]) < 0) return SW_E_CUDA;
            // a view's window stays a round deep (16 pending events per chain) however few warps it has: they loop
            if (round_batch_prep(x, first[v], n[v], G, 16, use_rc, Rv[v], Qv[v]) < 0) { e->err = x->err; return SW_E_CUDA; }
            Qv[v].slog = nullptr;                               // (the step log is for one cluster at a time)
            if (follow(x, x->stream.get(), e->stream.get()) < 0) { e->err = x->err; return SW_E_CUDA; }
        }
        CK(cudaMemcpyAsync(e->d_views.get() + v0, Rv.data() + v0, sizeof(RbParams) * nv, cudaMemcpyHostToDevice, e->stream.get()));
        {
            Span sp(e, e->stream.get(), SpanCat::rounds);
            if (use_rc) CK(cudaMemcpyAsync(e->d_rcviews.get() + v0, Qv.data() + v0, sizeof(RcParams) * nv, cudaMemcpyHostToDevice, e->stream.get()));
            if (round_kernels<NC, UNIT>(e, (const RbParams *)e->d_views.get() + v0, (const RcParams *)e->d_rcviews.get() + v0, nv, G, use_rc, e->stream.get()) < 0)
                return SW_E_CUDA;
            count_round_kernels(e, use_rc);
        }
        CK(cudaStreamSynchronize(e->stream.get()));       // (Rv is reused by the next group; the views' finish kernels follow)
        for (int v = v0; v < v0 + nv; v++) {
            if (round_batch_finish<NC>(engines[v], Rv[v]) < 0) return SW_E_CUDA;
            divided(engines[v], n[v]);
        }
    }
    return SW_OK;
}

// sw_verify_events' refusals, before anything runs: keys, creators, offsets (n + 1 of them, from 0, monotone)
int verify_args(sw_engine *e, const char *what, int n, const int32_t *creator, const int64_t *msg_off,
                const int64_t *pre_off, bool check_creators) {
    if (!e->have_keys) return fail(e, SW_E_ARG, "%s: no member keys (sw_set_member_keys)", what);
    for (const int64_t *off : {msg_off, pre_off}) {
        if (off[0] != 0) return fail(e, SW_E_ARG, "%s: offsets must start at 0", what);
        for (int i = 0; i < n; i++)
            if (off[i + 1] < off[i]) return fail(e, SW_E_ARG, "%s: offsets are not monotone at %d", what, i);
    }
    if (check_creators)
        for (int i = 0; i < n; i++)
            if (creator[i] < 0 || creator[i] >= e->M) return fail(e, SW_E_ARG, "%s: creator %d of event %d out of range", what, creator[i], i);
    return 0;
}

// Verify events sel[0..n) of the caller's columns (sel null: events 0..n), flags into flags_out[0..n): the columns
// are packed into one pinned block and go over in one copy; both kernels run on the compute stream; one sync.
// Keys: event j's creator is a member of views[set[j]], one of nviews engines on the device of e (set null: of e); the
// views' key sets then go over in the same block, and the kernels read event j's from there.
int verify_run(sw_engine *e, int n, const int *sel, const int *set, sw_engine *const *views, int nviews,
               const int32_t *creator, const uint8_t *sig, const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre,
               const int64_t *pre_off, const uint8_t *ids, uint8_t *flags_out) {
    if (n == 0) return SW_OK;
    auto src = [&](int j) { return sel ? sel[j] : j; };
    size_t mbytes = 0, pbytes = 0;
    for (int j = 0; j < n; j++) {
        mbytes += (size_t)(msg_off[src(j) + 1] - msg_off[src(j)]);
        pbytes += (size_t)(pre_off[src(j) + 1] - pre_off[src(j)]);
    }
    // the block: creator | set | key sets | msg_off | pre_off | sig | ids | msg | pre, each section 256-byte aligned
    // (set and key sets are empty for one engine's keys)
    const size_t nsets = set ? (size_t)nviews : 0;
    const size_t o_set = align256(sizeof(int32_t) * n), o_ks = o_set + align256(set ? sizeof(int32_t) * n : 0);
    const size_t o_moff = o_ks + align256(sizeof(KeySet) * nsets), o_poff = o_moff + align256(sizeof(int64_t) * (n + 1));
    const size_t o_sig = o_poff + align256(sizeof(int64_t) * (n + 1)), o_ids = o_sig + align256((size_t)64 * n);
    const size_t o_msg = o_ids + align256((size_t)32 * n), o_pre = o_msg + align256(mbytes), bytes = o_pre + pbytes;
    const size_t want = std::max(bytes, 2 * e->d_vin.cap());
    if (grow(e, bytes, e->d_vin.cap(), sized(e->d_vin, want), sized(e->h_vin, want)) < 0) return SW_E_CUDA;
    const size_t wn = std::max((size_t)n, 2 * e->d_vflags.cap());
    if (grow(e, n, e->d_vflags.cap(), sized(e->d_vflags, wn), sized(e->h_vflags, wn), sized(e->d_vk, 32 * wn)) < 0) return SW_E_CUDA;
    uint8_t *h = e->h_vin.get();
    int32_t *cr = (int32_t *)h, *vs = (int32_t *)(h + o_set);
    KeySet *ks = (KeySet *)(h + o_ks);
    for (size_t v = 0; v < nsets; v++) ks[v] = KeySet{views[v]->d_vkeys.get(), views[v]->d_vkey_ok.get(), views[v]->d_vatab.get()};
    int64_t *mo = (int64_t *)(h + o_moff), *po = (int64_t *)(h + o_poff);
    mo[0] = po[0] = 0;
    for (int j = 0; j < n; j++) {
        const int i = src(j);
        const int64_t ml = msg_off[i + 1] - msg_off[i], pl = pre_off[i + 1] - pre_off[i];
        cr[j] = creator[i];
        if (set) vs[j] = set[j];
        memcpy(h + o_sig + (size_t)64 * j, sig + (size_t)64 * i, 64);
        memcpy(h + o_ids + (size_t)32 * j, ids + (size_t)32 * i, 32);
        if (ml) memcpy(h + o_msg + mo[j], msg + msg_off[i], ml);
        if (pl) memcpy(h + o_pre + po[j], pre + pre_off[i], pl);
        mo[j + 1] = mo[j] + ml;
        po[j + 1] = po[j] + pl;
    }
    cudaStream_t st = e->stream.get();
    uint8_t *d = e->d_vin.get();
    CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st));
    const int32_t *dcr = (const int32_t *)d, *dset = set ? (const int32_t *)(d + o_set) : nullptr;
    const int64_t *dmo = (const int64_t *)(d + o_moff), *dpo = (const int64_t *)(d + o_poff);
    const int nb_hash = (int)std::min<long>((n + 255) / 256, 8L * e->n_sm);
    const int nb_curve = (int)std::min<long>((n + 127) / 128, 16L * e->n_sm);
    if (set) {
        const KeySet *dks = (const KeySet *)(d + o_ks);
        k_verify_hash<<<nb_hash, 256, 0, st>>>(n, dcr, dset, dks, d + o_sig, d + o_msg, dmo, d + o_pre, dpo, d + o_ids,
                                               e->d_vk.get(), e->d_vflags.get());
        k_verify_curve<<<nb_curve, 128, 0, st>>>(n, dcr, dset, dks, d + o_sig, e->d_vbtab.get(), e->d_vk.get(), e->d_vflags.get());
    } else {
        const KeySet K{e->d_vkeys.get(), e->d_vkey_ok.get(), e->d_vatab.get()};
        k_verify_hash<<<nb_hash, 256, 0, st>>>(n, dcr, dset, K, d + o_sig, d + o_msg, dmo, d + o_pre, dpo, d + o_ids,
                                               e->d_vk.get(), e->d_vflags.get());
        k_verify_curve<<<nb_curve, 128, 0, st>>>(n, dcr, dset, K, d + o_sig, e->d_vbtab.get(), e->d_vk.get(), e->d_vflags.get());
    }
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(e->h_vflags.get(), e->d_vflags.get(), n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    memcpy(flags_out, e->h_vflags.get(), n);
    e->stats.kernel_launches += 2;
    e->stats.h2d_bytes += (i64)bytes;
    e->stats.d2h_bytes += n;
    return SW_OK;
}

// Node.add_event for B node-views whose arguments are checked (sw_batch_append, sw_batch_ingest_verified): view v
// appends rows offsets[v] .. offsets[v+1] of the concatenated columns.  Every view is validated as sw_append validates
// it; the views of at most STAGE_EVENTS events go over packed in ONE block (their parameters first) and are scattered by
// ONE k_unpack, on the first engine's copy stream; larger views make the copies their sw_append makes, on their own copy
// streams.  rc_out[v] is view v's code; returns the first failing view's code (SW_E_CUDA: the call stopped there).
int append_views(sw_engine *const *engines, int B, const int *offsets, const int32_t *p0, const int32_t *p1,
                 const int32_t *creator, const double *t, const uint8_t *sig, int32_t *rc_out) {
    sw_engine *e = engines[0];
    // 1. every view's checks; a view that fails them keeps its state and its error
    std::vector<int> packed;
    size_t bytes = 0;
    int first_err = SW_OK;
    for (int v = 0; v < B; v++) {
        sw_engine *x = engines[v];
        const int o = offsets[v], n = offsets[v + 1] - o;
        int r = n > 0 ? append_validate(x, n, p0 + o, p1 + o, creator + o) : SW_OK;
        rc_out[v] = r;
        if (r < 0) { if (first_err == SW_OK) first_err = r; continue; }
        if (n == 0) continue;
        if (n <= sw_engine::STAGE_EVENTS) { packed.push_back(v); bytes += (unpack_bytes(n) + 15) & ~(size_t)15; }
        else if (append_copy(x, n, p0 + o, p1 + o, creator + o, t + o, sig + (size_t)64 * o) < 0 || append_commit(x, n, x->copy_stream.get()) < 0) {
            e->err = x->err;
            return SW_E_CUDA;
        }
    }
    if (packed.empty()) return first_err;
    bytes += align256(sizeof(UnpackParams) * packed.size());
    // 2. the packed views: one slot of the first engine's ring, one copy, one scatter kernel
    const int si = stage_slot(e, bytes);
    if (si < 0) return si;
    uint8_t *hs = e->h_stage.get() + e->stage_bytes() * si, *ds = e->d_stage.get() + e->stage_bytes() * si;
    UnpackParams *U = reinterpret_cast<UnpackParams *>(hs);
    size_t off = align256(sizeof(UnpackParams) * packed.size());
    for (size_t i = 0; i < packed.size(); i++) {
        sw_engine *x = engines[packed[i]];
        const int o = offsets[packed[i]], n = offsets[packed[i] + 1] - o;
        U[i] = append_pack(x, n, p0 + o, p1 + o, creator + o, t + o, sig + (size_t)64 * o, hs + off, ds + off);
        off += (unpack_bytes(n) + 15) & ~(size_t)15;
    }
    if (unpack_staged(e, si, off, reinterpret_cast<const UnpackParams *>(ds), (int)packed.size()) < 0) return SW_E_CUDA;
    // each view's pending-append event comes from its own pool (wait_appends returns it there)
    for (int v : packed)
        if (append_commit(engines[v], offsets[v + 1] - offsets[v], e->copy_stream.get()) < 0) { e->err = engines[v]->err; return SW_E_CUDA; }
    return first_err;
}

}  // namespace

extern "C" {

int sw_version(void) { return 208; }

const char *sw_last_error(const sw_engine *e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int sw_create(int M, int capacity_events, const int64_t *stake, int coin_period, int device, sw_engine **out) {
    bool force_wide = false;                           // SW_FORCE_WIDE=1: the any-M kernels at M <= 64 too
    if (const char *v = getenv("SW_FORCE_WIDE")) force_wide = atoi(v) != 0;
    return create(M, capacity_events, stake, coin_period, device, M > 64 || force_wide, out);
}

void sw_destroy(sw_engine *e) {
    if (!e) return;
    cudaSetDevice(e->device);
    wait_appends(e, -1);
    sync_streams(e);
    fold_spans(e);
    if (e->d_sk.get()) {            // the signing key does not outlive the engine in freed device memory
        cudaMemsetAsync(e->d_sk.get(), 0, e->d_sk.cap(), e->stream.get());
        cudaStreamSynchronize(e->stream.get());
    }
    delete e;
}

int sw_reset(sw_engine *e) {
    if (!e) return SW_E_ARG;
    CK(cudaSetDevice(e->device));
    e->h_creator.clear();
    e->ids.clear();
    e->id_of.clear();
    e->h_stale_cum.assign(1, 0);
    int rc = reset_state(e);
    memset(&e->stats, 0, sizeof e->stats);
    return rc;
}

int sw_rewind(sw_engine *e) {
    if (!e) return SW_E_ARG;
    CK(cudaSetDevice(e->device));
    return reset_state(e, true);
}

int sw_event_record(sw_engine *e, int slot) {
    if (!e || slot < 0 || slot >= 16) return fail(e, SW_E_ARG, "bad event slot");
    CK(cudaSetDevice(e->device));
    if (!e->user_ev[slot].get()) CK(e->user_ev[slot].create(true));
    CK(cudaEventRecord(e->user_ev[slot].get(), e->stream.get()));
    return SW_OK;
}

int sw_event_elapsed_ms(sw_engine *e, int a, int b, double *ms_out) {
    if (!e || a < 0 || a >= 16 || b < 0 || b >= 16 || !ms_out || !e->user_ev[a].get() || !e->user_ev[b].get())
        return fail(e, SW_E_ARG, "bad event slot");
    CK(cudaSetDevice(e->device));
    CK(cudaEventSynchronize(e->user_ev[b].get()));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e->user_ev[a].get(), e->user_ev[b].get()));
    *ms_out = ms;
    return SW_OK;
}

int sw_append(sw_engine *e, int n, const int32_t *p0, const int32_t *p1, const int32_t *creator,
              const double *t, const uint8_t *sig) {
    if (!e || n < 0 || (n > 0 && (!p0 || !p1 || !creator || !t || !sig))) return fail(e, SW_E_ARG, "bad argument");
    if (n == 0) return SW_OK;
    if ((i64)e->n_events + n > e->cap) return fail(e, SW_E_CAPACITY, "capacity_events=%d exceeded", e->cap);
    CK(cudaSetDevice(e->device));
    int rc = append_validate(e, n, p0, p1, creator);
    if (rc < 0) return rc;
    // The copies go to their own stream: they touch only the new rows, so they overlap the kernels of
    // earlier chunks still running on the compute stream; later compute work waits for them.
    if (n <= sw_engine::STAGE_EVENTS) {
        // a handful of events: pack the eight columns into one pinned block, one copy, one scatter kernel
        const int si = stage_slot(e, unpack_bytes(n));
        if (si < 0) return si;
        const UnpackParams U = append_pack(e, n, p0, p1, creator, t, sig, e->h_stage.get() + e->stage_bytes() * si, e->d_stage.get() + e->stage_bytes() * si);
        if (unpack_staged(e, si, unpack_bytes(n), U, 1) < 0) return SW_E_CUDA;
    } else if (append_copy(e, n, p0, p1, creator, t, sig) < 0) return SW_E_CUDA;
    return append_commit(e, n, e->copy_stream.get());
}

// Node.add_event for B node-views in one call (append_views)
int sw_batch_append(sw_engine *const *engines, int B, const int *offsets, const int32_t *p0, const int32_t *p1,
                    const int32_t *creator, const double *t, const uint8_t *sig, int32_t *rc_out) {
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    if (!e || !offsets || !rc_out) return fail(e, SW_E_ARG, "bad argument");
    int rc = check_views(engines, B, "sw_batch_append", false);
    if (rc < 0) return rc;
    if (offsets[0] < 0) return fail(e, SW_E_ARG, "sw_batch_append: offsets[0] = %d", offsets[0]);
    for (int v = 0; v < B; v++)
        if (offsets[v + 1] < offsets[v])
            return fail(e, SW_E_ARG, "sw_batch_append: offsets[%d] = %d > offsets[%d] = %d", v, offsets[v], v + 1, offsets[v + 1]);
    if (offsets[B] > offsets[0] && (!p0 || !p1 || !creator || !t || !sig)) return fail(e, SW_E_ARG, "bad argument");
    CK(cudaSetDevice(e->device));
    return append_views(engines, B, offsets, p0, p1, creator, t, sig, rc_out);
}

int sw_divide_rounds(sw_engine *e, int first, int n) {
    if (!e || n < 0) return fail(e, SW_E_ARG, "bad argument");
    if (n == 0) return SW_OK;
    if (first != e->n_divided) return fail(e, SW_E_ARG, "divide_rounds: first=%d but %d events are divided (events must arrive in order)", first, e->n_divided);
    if (first + n > e->n_events) return fail(e, SW_E_KEY, "divide_rounds: events [%d,%d) not appended", first, first + n);
    CK(cudaSetDevice(e->device));
    const bool ahead = ahead_path(e, n);
    if (!ahead && rs_drain(e) < 0) return SW_E_CUDA;
    if (stream_path(e, first, n)) {
        if (wait_appends(e, first + n) < 0 || stream_kernel(e, stream_params(e, first, n), 1) < 0) return SW_E_CUDA;
        return stream_divided(e, n);         // (it wrote can_see rows and the carry heads on the compute stream)
    }
    // rows behind by more than one more call (the first call after sw_rewind in the resident pattern): the ahead path
    // scans the call's own rows first, so that its piece starts before the rest are scanned
    const int scan_from = ahead && first + n > e->n_rowed && e->n_events - (first + n) >= n ? e->n_rowed : -1;
    int rc = rows_ready(e, first, n, scan_from >= 0 ? first + n : -1);
    if (rc < 0) return rc;
    {
        Span sp(e, e->stream.get(), SpanCat::divide);
        rc = ahead ? SW_NCU(e, divide_ahead, e, first, n, scan_from)
           : e->wide ? SW_NJ(divide_rounds_wide, e, first, n) : SW_NCU(e, divide_round_batch, e, first, n, sp);
        if (rc < 0) return rc;
    }
    divided(e, n);
    return SW_OK;
}

// Node.divide_rounds for B independent node-views at once: every view takes the path its single call would take.  The
// views whose call takes the one-launch path join ONE k_stream_divide launch (any M, any stakes); the others go
// through chunk_views.
int sw_batch_divide_rounds(sw_engine *const *engines, int B, const int *first, const int *n) {
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    if (!e || !first || !n) return fail(e, SW_E_ARG, "bad argument");
    int rc = check_views(engines, B, "sw_batch_divide_rounds", true);
    if (rc < 0) return rc;
    std::vector<sw_engine *> sv, cv;                  // the views on the streaming path, and on the chunk path
    std::vector<int> sn, cfirst, cn;
    for (int v = 0; v < B; v++) {
        sw_engine *x = engines[v];
        if (n[v] <= 0 || first[v] != x->n_divided || first[v] + n[v] > x->n_events)
            return fail(e, SW_E_ARG, "sw_batch_divide_rounds: view %d: bad range [%d,%d)", v, first[v], first[v] + n[v]);
        if (stream_path(x, first[v], n[v])) { sv.push_back(x); sn.push_back(n[v]); }
        else { cv.push_back(x); cfirst.push_back(first[v]); cn.push_back(n[v]); }
    }
    for (sw_engine *x : cv)
        if (x->wide || x->unit != cv[0]->unit)
            return fail(e, SW_E_UNSUPPORTED, "sw_batch_divide_rounds: views whose calls bring more than %d events must be M <= 64 engines of one stake shape", sw_engine::STREAM_N);
    CK(cudaSetDevice(e->device));
    const int S = (int)sv.size();
    if (S > 0) {
        std::vector<StreamParams> Sv(S);
        for (int i = 0; i < S; i++) {
            sw_engine *x = sv[i];
            if (wait_appends(x, x->n_divided + sn[i]) < 0) { e->err = x->err; return SW_E_CUDA; }
            Sv[i] = stream_params(x, x->n_divided, sn[i]);
        }
        if (views_enter(e, sv.data(), S) < 0) return SW_E_CUDA;
        if (grow(e, S, e->d_stviews.cap(), sized(e->d_stviews, S)) < 0) return SW_E_CUDA;
        CK(cudaMemcpyAsync(e->d_stviews.get(), Sv.data(), sizeof(StreamParams) * S, cudaMemcpyHostToDevice, e->stream.get()));
        e->stats.h2d_bytes += sizeof(StreamParams) * S;
        if (stream_kernel(e, (const StreamParams *)e->d_stviews.get(), S) < 0) return SW_E_CUDA;
        // each view's later work runs after the batch: no copy, no host synchronisation
        if (views_resume(e, sv.data(), S) < 0) return SW_E_CUDA;
        for (int i = 0; i < S; i++)
            if (stream_divided(sv[i], sn[i]) < 0) { e->err = sv[i]->err; return SW_E_CUDA; }
    }
    if (!cv.empty()) return SW_NCU(cv[0], chunk_views, e, cv.data(), (int)cv.size(), cfirst.data(), cn.data());
    return SW_OK;
}

int sw_decide_fame(sw_engine *e, int32_t *new_c_out, int cap) {
    if (!e || cap < 0 || (cap > 0 && !new_c_out)) return fail(e, SW_E_ARG, "bad argument");
    CK(cudaSetDevice(e->device));
    if (e->n_divided == 0) return fail(e, SW_E_ARG, "decide_fame: no witnesses yet (max() of an empty dict, swirld.py:225)");
    {
        Span sp(e, e->stream.get(), SpanCat::fame);
        fame_kernels(e, fame_params(e), 1);
        CK(cudaGetLastError());
    }
    const int spec = fame_spec(e);
    CK(cudaMemcpyAsync(e->h_scal.get(), e->d_scal.get(), sizeof(int32_t) * (SC_COUNT + spec), cudaMemcpyDeviceToHost, e->stream.get()));
    CK(cudaStreamSynchronize(e->stream.get()));
    if (e->spans.size() >= 256) fold_spans(e);         // (the timings are read in sw_sync / sw_stats; not on every call)
    e->stats.d2h_bytes += sizeof(int32_t) * (SC_COUNT + spec);
    int r;
    const int rc = fame_result(e, new_c_out, cap, r);
    return rc < 0 ? rc : r;
}

int sw_find_order(sw_engine *e, const int32_t *new_c, int n) {
    return sw_find_order_out(e, new_c, n, nullptr, nullptr, nullptr, 0);
}

int sw_find_order_out(sw_engine *e, const int32_t *new_c, int n, int32_t *ev_out, double *ts_out, int32_t *rr_out, int cap) {
    if (!e || n < 0 || (n > 0 && !new_c) || cap < 0 || (cap > 0 && (!ev_out || !ts_out || !rr_out)))
        return fail(e, SW_E_ARG, "bad argument");
    const bool want = ev_out != nullptr;               // (sw_find_order: the count only)
    if (want && cap < e->n_divided - e->n_tx)
        return fail(e, SW_E_ARG, "find_order: cap=%d < %d events it may order", cap, e->n_divided - e->n_tx);
    if (n == 0) return 0;
    CK(cudaSetDevice(e->device));
    std::vector<int32_t> rs(new_c, new_c + n);
    int bad;
    if (!sort_rounds(e, rs.data(), n, bad)) return fail(e, SW_E_KEY, "find_order: unknown round %d", bad);
    if (order_scratch(e, n) < 0) return SW_E_CUDA;
    CK(cudaMemcpyAsync(e->d_rounds_in.get(), rs.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, e->stream.get()));
    OrderParams P = order_params(e, n, e->d_rounds_in.get());
    P.out_n = want ? order_spec(e) : 0;
    {
        Span sp(e, e->stream.get(), SpanCat::order);
        order_kernels(e, P, 1, n);
        CK(cudaGetLastError());
    }
    const size_t bytes = sizeof(int32_t) * (SC_COUNT + 4 * (size_t)P.out_n);
    CK(cudaMemcpyAsync(e->h_scal.get(), e->d_scal.get(), bytes, cudaMemcpyDeviceToHost, e->stream.get()));
    CK(cudaStreamSynchronize(e->stream.get()));      // (rs, the host vector of the rounds, was consumed by the copy above)
    fold_spans(e);
    e->stats.h2d_bytes += sizeof(int32_t) * n;
    e->stats.d2h_bytes += bytes;
    const int base = e->n_tx;
    const int r = order_result(e);
    if (r <= 0 || !want) return r;
    const int rest = order_output(e, e->stream.get(), base, r, reinterpret_cast<const OrderOut *>(e->h_scal.get() + SC_COUNT), P.out_n,
                                  ev_out, ts_out, rr_out);
    if (rest < 0) return rest;
    if (rest > 0) {
        CK(cudaStreamSynchronize(e->stream.get()));
        e->stats.d2h_bytes += (2 * sizeof(int32_t) + sizeof(double)) * (size_t)rest;
    }
    return r;
}

// Node.decide_fame for B node-views in one call: the fame kernels of every view side by side in one grid (blockIdx.y =
// view), then the scalars and the first new rounds of all views back in one copy.
int sw_batch_decide_fame(sw_engine *const *engines, int B, int32_t *new_c_out, int cap, int32_t *count_out) {
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    if (!e || cap < 0 || (cap > 0 && !new_c_out) || !count_out) return fail(e, SW_E_ARG, "bad argument");
    int rc = check_views(engines, B, "sw_batch_decide_fame", true);
    if (rc < 0) return rc;
    for (int v = 0; v < B; v++)
        if (engines[v]->n_divided == 0)
            return fail(e, SW_E_ARG, "sw_batch_decide_fame: view %d: no witnesses yet (max() of an empty dict, swirld.py:225)", v);
    CK(cudaSetDevice(e->device));
    const int S = SC_COUNT + FAME_SPEC;                // per view: the scalars and the new rounds sw_decide_fame copies
    const size_t pbytes = align256(sizeof(FameParams) * B), sbytes = sizeof(int32_t) * (size_t)S * B;
    if (views_buffer(e, pbytes + sbytes) < 0) return SW_E_CUDA;
    FameParams *hP = reinterpret_cast<FameParams *>(e->h_vbuf.get());
    for (int v = 0; v < B; v++) hP[v] = fame_params(engines[v]);
    const FameParams *Pv = reinterpret_cast<const FameParams *>(e->d_vbuf.get());
    int32_t *d_st = reinterpret_cast<int32_t *>(e->d_vbuf.get() + pbytes), *h_st = reinterpret_cast<int32_t *>(e->h_vbuf.get() + pbytes);
    if (views_enter(e, engines, B) < 0) return SW_E_CUDA;
    CK(cudaMemcpyAsync(e->d_vbuf.get(), e->h_vbuf.get(), sizeof(FameParams) * B, cudaMemcpyHostToDevice, e->stream.get()));
    e->stats.h2d_bytes += sizeof(FameParams) * B;
    {
        Span sp(e, e->stream.get(), SpanCat::fame);
        fame_kernels(e, Pv, B);
        k_views_gather<<<B, 256, 0, e->stream.get()>>>(Pv, d_st, S);
        CK(cudaGetLastError());
        e->stats.kernel_launches += 1;
    }
    if (views_leave(e, engines, B, h_st, d_st, sbytes) < 0) return SW_E_CUDA;
    if (e->spans.size() >= 256) fold_spans(e);
    int first_err = SW_OK;
    for (int v = 0; v < B; v++) {
        sw_engine *x = engines[v];
        memcpy(x->h_scal.get(), h_st + (size_t)S * v, sizeof(int32_t) * (SC_COUNT + fame_spec(x)));
        int r;
        if (fame_result(x, new_c_out + (size_t)cap * v, cap, r) < 0) { e->err = x->err; return SW_E_CUDA; }
        count_out[v] = r;
        if (r < 0 && first_err == SW_OK) first_err = r;
    }
    return first_err;
}

// Node.find_order for B node-views in one call: the five order kernels of every view with rounds to order side by side
// (blockIdx.y = view), the views' parameters and rounds in one copy there, their scalars in one copy back.
int sw_batch_find_order(sw_engine *const *engines, int B, const int32_t *new_c, const int *offsets, int32_t *count_out) {
    return sw_batch_find_order_out(engines, B, new_c, offsets, count_out, nullptr, nullptr, nullptr, nullptr, 0);
}

int sw_batch_find_order_out(sw_engine *const *engines, int B, const int32_t *new_c, const int *offsets, int32_t *count_out,
                            int32_t *ev_out, double *ts_out, int32_t *rr_out, int *out_offsets, int cap) {
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    const bool want = out_offsets != nullptr;          // (sw_batch_find_order: the counts only)
    if (!e || !offsets || !count_out || cap < 0 || (want && cap > 0 && (!ev_out || !ts_out || !rr_out)))
        return fail(e, SW_E_ARG, "bad argument");
    int rc = check_views(engines, B, "sw_batch_find_order", true);
    if (rc < 0) return rc;
    if (offsets[0] < 0) return fail(e, SW_E_ARG, "sw_batch_find_order: offsets[0] = %d", offsets[0]);
    for (int v = 0; v < B; v++)
        if (offsets[v + 1] < offsets[v])
            return fail(e, SW_E_ARG, "sw_batch_find_order: offsets[%d] = %d > offsets[%d] = %d", v, offsets[v], v + 1, offsets[v + 1]);
    const int total = offsets[B] - offsets[0];
    if (total > 0 && !new_c) return fail(e, SW_E_ARG, "bad argument");
    std::vector<int32_t> rs(total);
    if (total > 0) std::copy(new_c + offsets[0], new_c + offsets[B], rs.begin());
    std::vector<sw_engine *> act;                      // the views with rounds to order
    std::vector<int> act_v;
    int maxn = 0;
    for (int v = 0; v < B; v++) {
        const int n = offsets[v + 1] - offsets[v];
        int bad;
        if (!sort_rounds(engines[v], rs.data() + (offsets[v] - offsets[0]), n, bad))
            return fail(e, SW_E_KEY, "sw_batch_find_order: view %d: unknown round %d", v, bad);
        if (n > 0) { act.push_back(engines[v]); act_v.push_back(v); maxn = std::max(maxn, n); }
    }
    // the output: every view's window is the largest of the active views' (one row length for the gather)
    int win = 0;
    if (want) {
        i64 need = 0;
        for (int v = 0; v < B; v++) need += engines[v]->n_divided - engines[v]->n_tx;
        if (need > cap) return fail(e, SW_E_ARG, "sw_batch_find_order: cap=%d < %lld events the views may order", cap, (long long)need);
        for (sw_engine *x : act) win = std::max(win, order_spec(x));
    }
    for (int v = 0; v < B; v++) count_out[v] = 0;
    if (want) for (int v = 0; v <= B; v++) out_offsets[v] = 0;
    const int A = (int)act.size();
    if (A == 0) return SW_OK;
    CK(cudaSetDevice(e->device));
    for (int i = 0; i < A; i++) if (order_scratch(act[i], offsets[act_v[i] + 1] - offsets[act_v[i]]) < 0) { e->err = act[i]->err; return SW_E_CUDA; }
    // [A parameter blocks][the rounds] go over in one copy; A rows of the scalars and the output window come back in one
    const int S = SC_COUNT + 4 * win;
    const size_t pbytes = sizeof(OrderParams) * A, inbytes = pbytes + sizeof(int32_t) * total, soff = align256(inbytes);
    const size_t sbytes = sizeof(int32_t) * (size_t)S * A;
    if (views_buffer(e, soff + sbytes) < 0) return SW_E_CUDA;
    OrderParams *hP = reinterpret_cast<OrderParams *>(e->h_vbuf.get());
    int32_t *h_rounds = reinterpret_cast<int32_t *>(e->h_vbuf.get() + pbytes);
    const int32_t *d_rounds = reinterpret_cast<const int32_t *>(e->d_vbuf.get() + pbytes);
    if (total > 0) memcpy(h_rounds, rs.data(), sizeof(int32_t) * total);
    for (int i = 0; i < A; i++) {
        const int v = act_v[i];
        hP[i] = order_params(act[i], offsets[v + 1] - offsets[v], d_rounds + (offsets[v] - offsets[0]));
        hP[i].out_n = win;
    }
    const OrderParams *Pv = reinterpret_cast<const OrderParams *>(e->d_vbuf.get());
    int32_t *d_st = reinterpret_cast<int32_t *>(e->d_vbuf.get() + soff), *h_st = reinterpret_cast<int32_t *>(e->h_vbuf.get() + soff);
    if (views_enter(e, act.data(), A) < 0) return SW_E_CUDA;
    CK(cudaMemcpyAsync(e->d_vbuf.get(), e->h_vbuf.get(), inbytes, cudaMemcpyHostToDevice, e->stream.get()));
    e->stats.h2d_bytes += inbytes;
    {
        Span sp(e, e->stream.get(), SpanCat::order);
        order_kernels(e, Pv, A, maxn);
        k_views_gather<<<A, win ? 256 : 32, 0, e->stream.get()>>>(Pv, d_st, S);
        CK(cudaGetLastError());
        e->stats.kernel_launches += 1;
    }
    if (views_leave(e, act.data(), A, h_st, d_st, sbytes) < 0) return SW_E_CUDA;
    fold_spans(e);
    int first_err = SW_OK;
    size_t rest = 0;
    int pos = 0, vn = 0;                               // view v's output is packed at pos (out_offsets[v] .. [v+1])
    for (int i = 0; i < A; i++) {
        sw_engine *x = act[i];
        memcpy(x->h_scal.get(), h_st + (size_t)S * i, sizeof(int32_t) * SC_COUNT);
        const int base = x->n_tx;
        const int r = order_result(x);
        count_out[act_v[i]] = r;
        if (r < 0 && first_err == SW_OK) first_err = r;
        if (!want) continue;
        for (; vn <= act_v[i]; vn++) out_offsets[vn] = pos;
        if (r <= 0) continue;
        const int k = order_output(x, e->stream.get(), base, r, reinterpret_cast<const OrderOut *>(h_st + (size_t)S * i + SC_COUNT),
                                   win, ev_out + pos, ts_out + pos, rr_out + pos);
        if (k < 0) { e->err = x->err; return k; }
        rest += k;
        pos += r;
    }
    if (want) for (; vn <= B; vn++) out_offsets[vn] = pos;
    if (rest > 0) {                                    // the views that ordered more than the window: one more synchronisation
        CK(cudaStreamSynchronize(e->stream.get()));
        e->stats.d2h_bytes += (2 * sizeof(int32_t) + sizeof(double)) * rest;
    }
    return first_err;
}

int sw_members(const sw_engine *e) { return e ? e->M : SW_E_ARG; }
int sw_n_events(const sw_engine *e) { return e ? e->n_events : SW_E_ARG; }
int sw_n_divided(const sw_engine *e) { return e ? e->n_divided : SW_E_ARG; }
int sw_n_transactions(const sw_engine *e) { return e ? e->n_tx : SW_E_ARG; }

int sw_sync(sw_engine *e) {
    if (!e) return SW_E_ARG;
    CK(cudaSetDevice(e->device));
    if (wait_appends(e, -1) < 0) return SW_E_CUDA;
    CK(cudaMemcpyAsync(e->h_scal.get(), e->d_scal.get(), sizeof(int32_t) * SC_COUNT, cudaMemcpyDeviceToHost, e->stream.get()));
    CK(cudaStreamSynchronize(e->stream.get()));
    fold_spans(e);
    return device_error(e);
}

int sw_max_round(sw_engine *e) {
    int rc = sw_sync(e);
    if (rc < 0) return rc;
    return e->h_scal.get()[SC_MAX_ROUND];
}

int sw_stats(sw_engine *e, sw_stats_t *out) {
    if (!e || !out) return SW_E_ARG;
    int rc = sw_sync(e);
    *out = e->stats;
    return rc;
}

#define GETTER(NAME, TYPE, SRC, LIMIT, WIDTH)                                                        \
    int NAME(sw_engine *e, int first, int n, TYPE *out) {                                            \
        if (!e || first < 0 || n < 0 || (n > 0 && !out)) return fail(e, SW_E_ARG, "bad argument");  \
        if (first + n > (LIMIT)) return fail(e, SW_E_KEY, #NAME ": [%d,%d) out of range", first, first + n); \
        if (n == 0) return SW_OK;                                                                    \
        CK(cudaSetDevice(e->device));                                                                \
        if (wait_appends(e, -1) < 0) return SW_E_CUDA;                                               \
        CK(cudaMemcpyAsync(out, (SRC) + (size_t)first * (WIDTH), sizeof(TYPE) * (size_t)n * (WIDTH), \
                           cudaMemcpyDeviceToHost, e->stream.get()));                                     \
        CK(cudaStreamSynchronize(e->stream.get()));                                                        \
        e->stats.d2h_bytes += sizeof(TYPE) * (size_t)n * (WIDTH);                                    \
        return SW_OK;                                                                                \
    }

GETTER(sw_get_round, int32_t, e->d_round.get(), e->n_divided, 1)
GETTER(sw_get_witness_flags, uint8_t, e->d_wit.get(), e->n_divided, 1)
GETTER(sw_get_famous, int8_t, e->d_famous_ev.get(), e->n_events, 1)
GETTER(sw_get_can_see, int32_t, e->d_row.get(), e->n_divided, e->M)
GETTER(sw_get_witness_table, int32_t, e->d_W.get(), e->Rcap, e->M)
GETTER(sw_get_transactions, int32_t, e->d_tx.get(), e->n_tx, 1)
GETTER(sw_get_consensus_times, double, e->d_tx_ts, e->n_tx, 1)
GETTER(sw_get_rounds_received, int32_t, e->d_tx_rr, e->n_tx, 1)
GETTER(sw_get_idx, int32_t, e->d_idx.get(), e->n_events, 1)

int sw_get_height(sw_engine *e, int first, int n, int32_t *out) {
    if (!e || first < 0 || n < 0 || (n > 0 && !out)) return fail(e, SW_E_ARG, "bad argument");
    if (first + n > e->n_events) return fail(e, SW_E_KEY, "sw_get_height: out of range");
    memcpy(out, e->h_height.get() + first, sizeof(int32_t) * n);
    return SW_OK;
}

int sw_get_consensus(sw_engine *e, int32_t *out, int cap) {
    if (!e || cap < 0) return fail(e, SW_E_ARG, "bad argument");
    int mr = sw_max_round(e);
    if (mr < -1) return mr;
    std::vector<uint8_t> flags((size_t)mr + 2);
    if (mr >= 0) {
        CK(cudaMemcpyAsync(flags.data(), e->d_consensus.get(), (size_t)mr + 1, cudaMemcpyDeviceToHost, e->stream.get()));
        CK(cudaStreamSynchronize(e->stream.get()));
        e->stats.d2h_bytes += mr + 1;
    }
    int cnt = 0;
    for (int r = 0; r <= mr; r++)
        if (flags[r]) { if (cnt < cap) out[cnt] = r; cnt++; }
    return cnt;
}

int sw_debug_counters(sw_engine *e, int64_t *out16, int clear) {
    if (!e || !out16) return SW_E_ARG;
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream.get()));
    if (e->rs.on) CK(cudaStreamSynchronize(e->rs.stream.get()));     // (the round stream's kernels count there too)
    CK(cudaMemcpy(out16, e->d_dbg.get(), sizeof(long long) * 16, cudaMemcpyDeviceToHost));
    if (clear) CK(cudaMemset(e->d_dbg.get(), 0, sizeof(long long) * 40));
    return SW_OK;
}

int sw_rc_step_log(sw_engine *e, uint32_t *out, int64_t cap_words, int clear) {
    if (!e || cap_words < 0 || (cap_words > 0 && !out)) return SW_E_ARG;
    if (!e->d_rcslog.get()) return 0;
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream.get()));
    if (e->rs.on) CK(cudaStreamSynchronize(e->rs.stream.get()));
    unsigned head[2];
    CK(cudaMemcpy(head, e->d_rcslog.get(), sizeof(head), cudaMemcpyDeviceToHost));
    const size_t words = std::min<size_t>((size_t)cap_words, RC_LOGH + (size_t)std::min(head[0], head[1]) * RC_CS * RC_NLOG);
    if (words) CK(cudaMemcpy(out, e->d_rcslog.get(), sizeof(unsigned) * words, cudaMemcpyDeviceToHost));
    if (clear) CK(cudaMemset(e->d_rcslog.get(), 0, sizeof(unsigned)));
    return (int)head[0];
}

int sw_flush_l2(sw_engine *e, int64_t bytes) {
    if (!e || bytes <= 0) return SW_E_ARG;
    CK(cudaSetDevice(e->device));
    if (grow(e, bytes, e->d_flush.cap(), sized(e->d_flush, bytes)) < 0) return SW_E_CUDA;
    CK(cudaMemsetAsync(e->d_flush.get(), 0x5a, (size_t)bytes, e->stream.get()));
    return SW_OK;
}

// ---- ingest: what Node.sync does between the wire and divide_rounds (swirld.py:129-136, utils.py:8-21), natively
namespace {
Id32 id_key(const uint8_t *p) { Id32 k; memcpy(k.data(), p, 32); return k; }

// What an ingest appends, decided before anything is appended: the accepted events' columns in parents-first order,
// and the input row each comes from
struct IngestPlan {
    std::vector<int32_t> p0, p1, cr, src;
    std::vector<double> t;
    std::vector<uint8_t> sig;
    int size() const { return (int)src.size(); }
};

// The plan of sw_ingest and sw_ingest_verified (and of each view of sw_batch_ingest_verified): `ok` (null: all) is a
// per-event verdict; a new event without it is skipped like an invalid one, and so is whatever depends on it.
// index_out gets the known ids' indices and -1 for the rest.  Nothing of the engine changes; the accepted events take
// the indices n_events, n_events + 1, ... in plan order.
int ingest_plan(sw_engine *e, int n, const uint8_t *ids, const uint8_t *p0_ids, const uint8_t *p1_ids,
                const int32_t *creator, const double *t, const uint8_t *sig, const uint8_t *ok, int32_t *index_out,
                IngestPlan &P) {
    const auto key = id_key;
    const Id32 zero{};
    // 1. which events are new, and where each new id sits in the batch
    std::unordered_map<Id32, int, Id32Hash> inbatch;
    inbatch.reserve((size_t)n * 2);
    for (int i = 0; i < n; i++) {
        const Id32 k = key(ids + (size_t)32 * i);
        auto it = e->ids.find(k);
        if (it != e->ids.end()) index_out[i] = it->second;
        else { index_out[i] = -1; inbatch.emplace(k, i); }       // (a duplicate id in the batch: the first one counts)
    }
    // 2. parents-first order of the new ones (iterative DFS; the edges are the parents that are in the batch)
    std::vector<int> order, state(n, 0);                           // 0 unseen, 1 on the stack, 2 done
    order.reserve(inbatch.size());
    std::vector<std::pair<int, int>> stack;
    auto parent_in_batch = [&](int i, int which) -> int {
        const Id32 k = key((which ? p1_ids : p0_ids) + (size_t)32 * i);
        if (k == zero) return -1;
        auto it = inbatch.find(k);
        return it == inbatch.end() ? -1 : it->second;
    };
    for (int r = 0; r < n; r++) {
        if (index_out[r] >= 0 || state[r] || inbatch.find(key(ids + (size_t)32 * r))->second != r) continue;
        stack.push_back({r, 0});
        state[r] = 1;
        while (!stack.empty()) {
            auto &[u, next] = stack.back();
            if (next < 2) {
                const int v = parent_in_batch(u, next++);
                if (v < 0 || state[v] == 2) continue;
                if (state[v] == 1) return fail(e, SW_E_ARG, "sw_ingest: the batch is not a DAG (utils.py:13)");
                state[v] = 1;
                stack.push_back({v, 0});
            } else { state[u] = 2; order.push_back(u); stack.pop_back(); }
        }
    }
    // 3. validate in that order against a scratch copy of the chain heads; what fails (and what hangs below it) is skipped
    std::vector<int32_t> head(e->h_head), bidx(n, -1), bcreator;
    int next_index = e->n_events;
    auto resolve = [&](int i, int which, int &out) -> bool {        // parent id -> arrival index (-1: no parent)
        const Id32 k = key((which ? p1_ids : p0_ids) + (size_t)32 * i);
        if (k == zero) { out = -1; return true; }
        auto g = e->ids.find(k);
        if (g != e->ids.end()) { out = g->second; return true; }
        auto b = inbatch.find(k);
        if (b != inbatch.end() && bidx[b->second] >= 0) { out = bidx[b->second]; return true; }
        return false;
    };
    auto creator_of = [&](int idx) { return idx < e->n_events ? e->h_creator[idx] : bcreator[idx - e->n_events]; };
    for (int i : order) {
        const int c = creator[i];
        int a, b;
        if ((ok && !ok[i]) || c < 0 || c >= e->M || !resolve(i, 0, a) || !resolve(i, 1, b)) continue;
        if (a < 0 && b < 0) { if (head[c] >= 0) continue; }                         // a second root: fork
        else if (a < 0 || b < 0 || creator_of(a) != c || creator_of(b) == c || head[c] != a) continue;   // swirld.py:104-108 + fork-free
        if (next_index >= e->cap) return fail(e, SW_E_CAPACITY, "capacity_events=%d exceeded", e->cap);
        bidx[i] = next_index++;
        head[c] = bidx[i];
        bcreator.push_back(c);
        P.p0.push_back(a); P.p1.push_back(b); P.cr.push_back(c); P.t.push_back(t[i]); P.src.push_back(i);
    }
    P.sig.resize((size_t)64 * P.size());
    for (int j = 0; j < P.size(); j++) memcpy(P.sig.data() + (size_t)64 * j, sig + (size_t)64 * P.src[j], 64);
    return SW_OK;
}

// After the plan's events were appended (they are the engine's last P.size()): enter their ids, and fill index_out
void ingest_commit(sw_engine *e, int n, const uint8_t *ids, const IngestPlan &P, int32_t *index_out) {
    const int base = e->n_events - P.size();
    if (e->id_of.size() < (size_t)e->n_events) e->id_of.resize(e->n_events, Id32{});
    for (int j = 0; j < P.size(); j++) {
        const Id32 k = id_key(ids + (size_t)32 * P.src[j]);
        e->ids.emplace(k, base + j);
        e->id_of[base + j] = k;
    }
    for (int i = 0; i < n; i++)
        if (index_out[i] < 0) { auto it = e->ids.find(id_key(ids + (size_t)32 * i)); index_out[i] = it == e->ids.end() ? -1 : it->second; }
}

// sw_ingest and sw_ingest_verified: the plan, ONE sw_append, the ids
int ingest(sw_engine *e, int n, const uint8_t *ids, const uint8_t *p0_ids, const uint8_t *p1_ids,
           const int32_t *creator, const double *t, const uint8_t *sig, const uint8_t *ok, int32_t *index_out) {
    IngestPlan P;
    int rc = ingest_plan(e, n, ids, p0_ids, p1_ids, creator, t, sig, ok, index_out, P);
    if (rc < 0) return rc;
    const int m = P.size();
    if (m > 0) {
        rc = sw_append(e, m, P.p0.data(), P.p1.data(), P.cr.data(), P.t.data(), P.sig.data());
        if (rc < 0) return rc;
        // (pageable sources: the copies are staged before sw_append returns, the vectors may go)
        CK(cudaStreamSynchronize(e->copy_stream.get()));
    }
    ingest_commit(e, n, ids, P, index_out);
    return m;
}

int ingest_views(sw_engine *const *engines, int B, const int *offsets, const uint8_t *ids, const uint8_t *p0_ids,
                 const uint8_t *p1_ids, const int32_t *creator, const double *t, const uint8_t *sig, const uint8_t *ok,
                 int32_t *index_out, int32_t *count_out);
}  // namespace

int sw_ingest(sw_engine *e, int n, const uint8_t *ids, const uint8_t *p0_ids, const uint8_t *p1_ids,
              const int32_t *creator, const double *t, const uint8_t *sig, int32_t *index_out) {
    if (!e || n < 0 || (n > 0 && (!ids || !p0_ids || !p1_ids || !creator || !t || !sig || !index_out))) return fail(e, SW_E_ARG, "bad argument");
    return ingest(e, n, ids, p0_ids, p1_ids, creator, t, sig, nullptr, index_out);
}

int sw_set_member_keys(sw_engine *e, const uint8_t *pk) {
    if (!e || !pk) return fail(e, SW_E_ARG, "bad argument");
    CK(cudaSetDevice(e->device));
    const size_t M = e->M;
    if (grow(e, M, e->d_vkey_ok.cap(), sized(e->d_vkeys, 32 * M), sized(e->d_vkey_ok, M), sized(e->d_vatab, swv::TAB * M)) < 0) return SW_E_CUDA;
    cudaStream_t st = e->stream.get();
    if (!e->have_base) {            // [1..15]B, from the base point's encoding, once per engine
        if (grow(e, swv::TAB, e->d_vbtab.cap(), sized(e->d_vbtab, swv::TAB)) < 0) return SW_E_CUDA;
        k_verify_tables<<<1, 32, 0, st>>>(1, nullptr, nullptr, e->d_vbtab.get());
        e->stats.kernel_launches += 1;
    }
    e->h_vkeys.assign(pk, pk + 32 * M);
    CK(cudaMemcpyAsync(e->d_vkeys.get(), pk, 32 * M, cudaMemcpyHostToDevice, st));
    k_verify_tables<<<(int)((M + 63) / 64), 64, 0, st>>>((int)M, e->d_vkeys.get(), e->d_vkey_ok.get(), e->d_vatab.get());
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    e->stats.kernel_launches += 1;
    e->stats.h2d_bytes += (i64)(32 * M);
    e->have_keys = e->have_base = true;
    return SW_OK;
}

int sw_verify_events(sw_engine *e, int n, const int32_t *creator, const uint8_t *sig,
                     const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off,
                     const uint8_t *ids, uint8_t *flags_out) {
    if (!e || n < 0 || (n > 0 && (!creator || !sig || !msg_off || !pre_off || !ids || !flags_out)))
        return fail(e, SW_E_ARG, "bad argument");
    CK(cudaSetDevice(e->device));
    if (n > 0 && ((!msg && msg_off[n] > 0) || (!pre && pre_off[n] > 0))) return fail(e, SW_E_ARG, "bad argument");
    const int64_t zero = 0;
    const int rc = verify_args(e, "sw_verify_events", n, creator, n ? msg_off : &zero, n ? pre_off : &zero, true);
    return rc < 0 ? rc : verify_run(e, n, nullptr, nullptr, nullptr, 0, creator, sig, msg, msg_off, pre, pre_off, ids, flags_out);
}

int sw_ingest_verified(sw_engine *e, int n, const uint8_t *ids, const uint8_t *p0_ids, const uint8_t *p1_ids,
                       const int32_t *creator, const double *t, const uint8_t *sig,
                       const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off,
                       int32_t *index_out) {
    if (!e || n < 0 || (n > 0 && (!ids || !p0_ids || !p1_ids || !creator || !t || !sig || !index_out || !msg_off || !pre_off)))
        return fail(e, SW_E_ARG, "bad argument");
    CK(cudaSetDevice(e->device));
    if (n > 0 && ((!msg && msg_off[n] > 0) || (!pre && pre_off[n] > 0))) return fail(e, SW_E_ARG, "bad argument");
    const int64_t zero = 0;
    int rc = verify_args(e, "sw_ingest_verified", n, creator, n ? msg_off : &zero, n ? pre_off : &zero, false);
    if (rc < 0) return rc;
    // the new ids (the first event of each, as ingest counts it) whose creator is a member: only they are verified; a
    // new event with another creator is skipped by ingest anyway
    std::vector<int> fresh;
    {
        std::unordered_map<Id32, int, Id32Hash> seen;
        for (int i = 0; i < n; i++) {
            const Id32 k = id_key(ids + (size_t)32 * i);
            if (e->ids.count(k) || !seen.emplace(k, i).second) continue;
            if (creator[i] >= 0 && creator[i] < e->M) fresh.push_back(i);
        }
    }
    std::vector<uint8_t> flags(fresh.size()), ok(n, 1);
    rc = verify_run(e, (int)fresh.size(), fresh.data(), nullptr, nullptr, 0, creator, sig, msg, msg_off, pre, pre_off, ids, flags.data());
    if (rc < 0) return rc;
    for (size_t j = 0; j < fresh.size(); j++) ok[fresh[j]] = flags[j] == 3;
    return ingest(e, n, ids, p0_ids, p1_ids, creator, t, sig, ok.data(), index_out);
}

// Node.sync's ingest for B node-views in one call.  Each view plans what its sw_ingest_verified would plan, but the
// events the views would verify go to the GPU once per distinct event, all in one block on the first engine's stream,
// and the accepted events of every view go over through append_views.
int sw_batch_ingest_verified(sw_engine *const *engines, int B, const int *offsets, const uint8_t *ids,
                             const uint8_t *p0_ids, const uint8_t *p1_ids, const int32_t *creator, const double *t,
                             const uint8_t *sig, const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre,
                             const int64_t *pre_off, int32_t *index_out, int32_t *count_out, int32_t *n_verified_out) {
    const char *what = "sw_batch_ingest_verified";
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    if (!e || !offsets || !count_out || !msg_off || !pre_off) return fail(e, SW_E_ARG, "bad argument");
    int rc = check_views(engines, B, what, false);
    if (rc < 0) return rc;
    for (int v = 0; v < B; v++)
        if (!engines[v]->have_keys) return fail(e, SW_E_ARG, "%s: view %d has no member keys (sw_set_member_keys)", what, v);
    if (offsets[0] < 0) return fail(e, SW_E_ARG, "%s: offsets[0] = %d", what, offsets[0]);
    for (int v = 0; v < B; v++)
        if (offsets[v + 1] < offsets[v])
            return fail(e, SW_E_ARG, "%s: offsets[%d] = %d > offsets[%d] = %d", what, v, offsets[v], v + 1, offsets[v + 1]);
    const int N = offsets[B];
    if (N > 0 && (!ids || !p0_ids || !p1_ids || !creator || !t || !sig || !index_out)) return fail(e, SW_E_ARG, "bad argument");
    rc = verify_args(e, what, N, creator, msg_off, pre_off, false);
    if (rc < 0) return rc;
    if ((!msg && msg_off[N] > 0) || (!pre && pre_off[N] > 0)) return fail(e, SW_E_ARG, "bad argument");
    CK(cudaSetDevice(e->device));

    // 1. the events each view would verify (new to the view, the first row of their id among the view's rows, a
    //    member's creator), merged across views when their verdict must be the same: the same key, and byte-identical
    //    id, signature, message and preimage.  Distinct event k is first seen at row rep[k] of view vset[k].
    std::vector<int> rep, vset, distinct(N, -1);                    // distinct[r]: row r's distinct event (-1: none)
    std::unordered_map<Id32, std::vector<int>, Id32Hash> by_id;      // id -> its distinct events
    auto span_eq = [](const uint8_t *base, const int64_t *off, int r, int q) {
        const int64_t len = off[r + 1] - off[r];
        return len == off[q + 1] - off[q] && (len == 0 || !memcmp(base + off[r], base + off[q], len));
    };
    auto same = [&](int r, int v, int k) {
        const int q = rep[k];
        return !memcmp(engines[v]->h_vkeys.data() + (size_t)32 * creator[r], engines[vset[k]]->h_vkeys.data() + (size_t)32 * creator[q], 32) &&
               !memcmp(sig + (size_t)64 * r, sig + (size_t)64 * q, 64) && span_eq(msg, msg_off, r, q) && span_eq(pre, pre_off, r, q);
    };
    for (int v = 0; v < B; v++) {
        const sw_engine *x = engines[v];
        std::unordered_set<Id32, Id32Hash> seen;
        for (int r = offsets[v]; r < offsets[v + 1]; r++) {
            const Id32 k = id_key(ids + (size_t)32 * r);
            if (x->ids.count(k) || !seen.insert(k).second || creator[r] < 0 || creator[r] >= x->M) continue;
            std::vector<int> &cands = by_id[k];
            int d = -1;
            for (int c : cands) if (same(r, v, c)) { d = c; break; }
            if (d < 0) { d = (int)rep.size(); rep.push_back(r); vset.push_back(v); cands.push_back(d); }
            distinct[r] = d;
        }
    }
    // 2. each distinct event once on the GPU
    std::vector<uint8_t> flags(rep.size());
    rc = verify_run(e, (int)rep.size(), rep.data(), vset.data(), engines, B, creator, sig, msg, msg_off, pre, pre_off, ids, flags.data());
    if (rc < 0) return rc;
    if (n_verified_out) *n_verified_out = (int32_t)rep.size();
    std::vector<uint8_t> ok(N, 1);
    for (int r = 0; r < N; r++) if (distinct[r] >= 0) ok[r] = flags[distinct[r]] == 3;
    return ingest_views(engines, B, offsets, ids, p0_ids, p1_ids, creator, t, sig, ok.data(), index_out, count_out);
}

namespace {
// The ingest of B node-views after their verdicts (sw_batch_ingest_verified, sw_batch_new_events): view v ingests rows
// offsets[v] .. offsets[v+1] as its sw_ingest_verified would with verdicts ok[row] (null: all accepted).
int ingest_views(sw_engine *const *engines, int B, const int *offsets, const uint8_t *ids, const uint8_t *p0_ids,
                 const uint8_t *p1_ids, const int32_t *creator, const double *t, const uint8_t *sig, const uint8_t *ok,
                 int32_t *index_out, int32_t *count_out) {
    sw_engine *e = engines[0];
    // 3. every view's plan with its verdicts; a view that fails keeps its state and its error, and appends nothing
    std::vector<IngestPlan> plans(B);
    std::vector<int> aoff(B + 1, 0);
    for (int v = 0; v < B; v++) {
        const int o = offsets[v], n = offsets[v + 1] - o;
        count_out[v] = ingest_plan(engines[v], n, ids + (size_t)32 * o, p0_ids + (size_t)32 * o, p1_ids + (size_t)32 * o,
                                   creator + o, t + o, sig + (size_t)64 * o, ok ? ok + o : nullptr, index_out + o, plans[v]);
        if (count_out[v] < 0) plans[v] = IngestPlan();
        aoff[v + 1] = aoff[v] + plans[v].size();
    }
    // 4. the accepted events, concatenated, through the path of sw_batch_append
    const int A = aoff[B];
    std::vector<int32_t> c_p0(A), c_p1(A), c_cr(A), arc(B);
    std::vector<double> c_t(A);
    std::vector<uint8_t> c_sig((size_t)64 * A);
    for (int v = 0; v < B; v++) {
        const IngestPlan &P = plans[v];
        const int o = aoff[v], m = P.size();
        std::copy_n(P.p0.data(), m, c_p0.data() + o); std::copy_n(P.p1.data(), m, c_p1.data() + o); std::copy_n(P.cr.data(), m, c_cr.data() + o);
        std::copy_n(P.t.data(), m, c_t.data() + o); std::copy_n(P.sig.data(), (size_t)64 * m, c_sig.data() + (size_t)64 * o);
    }
    if (A > 0 && append_views(engines, B, aoff.data(), c_p0.data(), c_p1.data(), c_cr.data(), c_t.data(), c_sig.data(), arc.data()) == SW_E_CUDA)
        return SW_E_CUDA;
    // (pageable sources: the large views' copies are staged once their copy streams are done, then the vectors may go)
    for (int v = 0; v < B; v++)
        if (aoff[v + 1] - aoff[v] > sw_engine::STAGE_EVENTS) CK(cudaStreamSynchronize(engines[v]->copy_stream.get()));
    // 5. the ids of what each view appended
    int first_err = SW_OK;
    for (int v = 0; v < B; v++) {
        if (count_out[v] >= 0 && arc[v] < 0) count_out[v] = arc[v];
        if (count_out[v] < 0) { if (first_err == SW_OK) first_err = count_out[v]; continue; }
        const int o = offsets[v];
        ingest_commit(engines[v], offsets[v + 1] - o, ids + (size_t)32 * o, plans[v], index_out + o);
        count_out[v] = plans[v].size();
    }
    return first_err;
}

// Zeros over n bytes of host memory that the compiler may not drop
void wipe(void *p, size_t n) {
    volatile uint8_t *q = static_cast<volatile uint8_t *>(p);
    for (size_t i = 0; i < n; i++) q[i] = 0;
}

// Calls of at most this many events sign with 8 lanes per event (k_sign_events<8>), larger ones with one (DESIGN §5)
constexpr int SIGN_SPLIT_N = 4096;

// sw_new_events' refusals, before anything runs: offsets (n + 1 of them, from 0, monotone) and sig_at in [0, len - 64]
int sign_args(sw_engine *e, const char *what, int n, const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre,
              const int64_t *pre_off, const int64_t *sig_at) {
    for (const int64_t *off : {msg_off, pre_off}) {
        if (off[0] != 0) return fail(e, SW_E_ARG, "%s: offsets must start at 0", what);
        for (int i = 0; i < n; i++)
            if (off[i + 1] < off[i]) return fail(e, SW_E_ARG, "%s: offsets are not monotone at %d", what, i);
    }
    for (int i = 0; i < n; i++)
        if (sig_at[i] < 0 || sig_at[i] > pre_off[i + 1] - pre_off[i] - 64)
            return fail(e, SW_E_ARG, "%s: sig_at %lld of event %d is outside its preimage", what, (long long)sig_at[i], i);
    if ((!msg && msg_off[n] > 0) || (!pre && pre_off[n] > 0)) return fail(e, SW_E_ARG, "%s: bad argument", what);
    return 0;
}

// Sign events 0..n and hash their preimages: the inputs go over in one pinned block, k_sign_events runs on the compute
// stream of e, the signatures and ids come back in one copy, one synchronisation.  Event j is signed by the key of
// views[set[j]] (set null: of e); the table is e's.
int sign_run(sw_engine *e, int n, const int *set, sw_engine *const *views, int nviews, const uint8_t *msg,
             const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off, const int64_t *sig_at, uint8_t *sig_out,
             uint8_t *ids_out) {
    if (n == 0) return SW_OK;
    const size_t nkeys = set ? (size_t)nviews : 1, mbytes = (size_t)msg_off[n], pbytes = (size_t)pre_off[n];
    // the block: set | keys | msg_off | pre_off | sig_at | msg | pre, each section 256-byte aligned
    const size_t o_keys = align256(set ? sizeof(int32_t) * n : 0), o_moff = o_keys + align256(sizeof(void *) * nkeys);
    const size_t o_poff = o_moff + align256(sizeof(int64_t) * (n + 1)), o_at = o_poff + align256(sizeof(int64_t) * (n + 1));
    const size_t o_msg = o_at + align256(sizeof(int64_t) * n), o_pre = o_msg + align256(mbytes), bytes = o_pre + pbytes;
    const size_t want = std::max(bytes, 2 * e->d_vin.cap());
    if (grow(e, bytes, e->d_vin.cap(), sized(e->d_vin, want), sized(e->h_vin, want)) < 0) return SW_E_CUDA;
    const size_t wn = std::max((size_t)96 * n, 2 * e->d_sout.cap());
    if (grow(e, (size_t)96 * n, e->d_sout.cap(), sized(e->d_sout, wn), sized(e->h_sout, wn)) < 0) return SW_E_CUDA;
    uint8_t *h = e->h_vin.get(), *d = e->d_vin.get();
    if (set) memcpy(h, set, sizeof(int32_t) * n);
    const uint8_t **keys = reinterpret_cast<const uint8_t **>(h + o_keys);
    for (size_t v = 0; v < nkeys; v++) keys[v] = (set ? views[v] : e)->d_sk.get();
    memcpy(h + o_moff, msg_off, sizeof(int64_t) * (n + 1));
    memcpy(h + o_poff, pre_off, sizeof(int64_t) * (n + 1));
    memcpy(h + o_at, sig_at, sizeof(int64_t) * n);
    if (mbytes) memcpy(h + o_msg, msg, mbytes);
    if (pbytes) memcpy(h + o_pre, pre, pbytes);
    cudaStream_t st = e->stream.get();
    CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st));
    const int32_t *dset = set ? reinterpret_cast<const int32_t *>(d) : nullptr;
    const uint8_t *const *dkeys = reinterpret_cast<const uint8_t *const *>(d + o_keys);
    const int64_t *dmo = reinterpret_cast<const int64_t *>(d + o_moff), *dpo = reinterpret_cast<const int64_t *>(d + o_poff);
    const int64_t *dat = reinterpret_cast<const int64_t *>(d + o_at);
    uint8_t *dsig = e->d_sout.get(), *dids = dsig + (size_t)64 * n;
    if (n <= SIGN_SPLIT_N)
        k_sign_events<8><<<(n + 15) / 16, 128, 0, st>>>(n, dset, dkeys, e->d_comb.get(), d + o_msg, dmo, d + o_pre, dpo, dat, dsig, dids);
    else
        k_sign_events<1><<<(int)std::min<long>((n + 127) / 128, 16L * e->n_sm), 128, 0, st>>>(n, dset, dkeys, e->d_comb.get(), d + o_msg,
                                                                                               dmo, d + o_pre, dpo, dat, dsig, dids);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(e->h_sout.get(), dsig, (size_t)96 * n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    memcpy(sig_out, e->h_sout.get(), (size_t)64 * n);
    memcpy(ids_out, e->h_sout.get() + (size_t)64 * n, (size_t)32 * n);
    e->stats.kernel_launches += 1;
    e->stats.h2d_bytes += (i64)bytes;
    e->stats.d2h_bytes += (i64)96 * n;
    return SW_OK;
}
}  // namespace

int sw_set_signing_key(sw_engine *e, int member, const uint8_t *sk) {
    const char *what = "sw_set_signing_key";
    if (!e || !sk) return fail(e, SW_E_ARG, "bad argument");
    if (!e->have_keys) return fail(e, SW_E_ARG, "%s: no member keys (sw_set_member_keys)", what);
    if (member < 0 || member >= e->M) return fail(e, SW_E_ARG, "%s: member %d out of range", what, member);
    if (memcmp(sk + 32, e->h_vkeys.data() + (size_t)32 * member, 32))
        return fail(e, SW_E_ARG, "%s: sk[32..64) is not member %d's key", what, member);
    CK(cudaSetDevice(e->device));
    cudaStream_t st = e->stream.get();
    if (grow(e, 1, e->d_sk.get() ? 1 : 0, sized(e->d_sk, sws::SK_BYTES)) < 0 ||
        grow(e, 1, e->d_skin.get() ? 1 : 0, sized(e->d_skin, 65), sized(e->h_skin, 65)) < 0)
        return SW_E_CUDA;
    if (!e->have_comb) {            // j 256^k B, from the base point's encoding, once per engine
        if (grow(e, 1, 0, sized(e->d_comb, sws::ROWS * sws::COLS)) < 0) return SW_E_CUDA;
        k_sign_table<<<1, 32, 0, st>>>(e->d_comb.get());
        CK(cudaGetLastError());
        e->stats.kernel_launches += 1;
        e->have_comb = true;
    }
    uint8_t *h = e->h_skin.get();
    memcpy(h, sk, 64);
    cudaError_t s = cudaMemcpyAsync(e->d_skin.get(), h, 64, cudaMemcpyHostToDevice, st);
    if (s == cudaSuccess) {
        k_sign_key<<<1, 32, 0, st>>>(e->d_skin.get(), e->d_comb.get(), e->d_sk.get(), e->d_skin.get() + 64);
        s = cudaGetLastError();
    }
    if (s == cudaSuccess) s = cudaMemcpyAsync(h + 64, e->d_skin.get() + 64, 1, cudaMemcpyDeviceToHost, st);
    const cudaError_t w = cudaMemsetAsync(e->d_skin.get(), 0, 64, st);
    if (s == cudaSuccess) s = w;
    if (s == cudaSuccess) s = cudaStreamSynchronize(st);
    wipe(h, 64);
    if (s != cudaSuccess) return fail(e, SW_E_CUDA, "%s: %s", what, cudaGetErrorString(s));
    e->stats.kernel_launches += 1;
    e->stats.h2d_bytes += 64;
    e->stats.d2h_bytes += 1;
    if (!h[64]) return fail(e, SW_E_ARG, "%s: [a]B of the seed does not encode to member %d's key", what, member);
    e->have_sign = true;
    e->sign_member = member;
    return SW_OK;
}

int sw_new_events(sw_engine *e, int n, const uint8_t *p0_ids, const uint8_t *p1_ids, const double *t,
                  const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off,
                  const int64_t *sig_at, uint8_t *sig_out, uint8_t *ids_out, int32_t *index_out) {
    const char *what = "sw_new_events";
    if (!e || n < 0 || (n > 0 && (!msg_off || !pre_off || !sig_at || !sig_out || !ids_out)) ||
        (n > 0 && index_out && (!p0_ids || !p1_ids || !t)))
        return fail(e, SW_E_ARG, "bad argument");
    if (!e->have_sign) return fail(e, SW_E_ARG, "%s: no signing key (sw_set_signing_key)", what);
    if (n == 0) return SW_OK;
    int rc = sign_args(e, what, n, msg, msg_off, pre, pre_off, sig_at);
    if (rc < 0) return rc;
    CK(cudaSetDevice(e->device));
    rc = sign_run(e, n, nullptr, nullptr, 0, msg, msg_off, pre, pre_off, sig_at, sig_out, ids_out);
    if (rc < 0 || !index_out) return rc;
    const std::vector<int32_t> creator(n, e->sign_member);
    return ingest(e, n, ids_out, p0_ids, p1_ids, creator.data(), t, sig_out, nullptr, index_out);
}

int sw_batch_new_events(sw_engine *const *engines, int B, const int *offsets, const uint8_t *p0_ids,
                        const uint8_t *p1_ids, const double *t, const uint8_t *msg, const int64_t *msg_off,
                        const uint8_t *pre, const int64_t *pre_off, const int64_t *sig_at, uint8_t *sig_out,
                        uint8_t *ids_out, int32_t *index_out, int32_t *count_out) {
    const char *what = "sw_batch_new_events";
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    if (!e || !offsets || !msg_off || !pre_off || (index_out && !count_out)) return fail(e, SW_E_ARG, "bad argument");
    int rc = check_views(engines, B, what, false, index_out != nullptr);
    if (rc < 0) return rc;
    for (int v = 0; v < B; v++)
        if (!engines[v]->have_sign) return fail(e, SW_E_ARG, "%s: view %d has no signing key (sw_set_signing_key)", what, v);
    if (offsets[0] != 0) return fail(e, SW_E_ARG, "%s: offsets[0] = %d", what, offsets[0]);
    for (int v = 0; v < B; v++)
        if (offsets[v + 1] < offsets[v])
            return fail(e, SW_E_ARG, "%s: offsets[%d] = %d > offsets[%d] = %d", what, v, offsets[v], v + 1, offsets[v + 1]);
    const int N = offsets[B];
    if (N > 0 && (!sig_at || !sig_out || !ids_out || (index_out && (!p0_ids || !p1_ids || !t))))
        return fail(e, SW_E_ARG, "bad argument");
    rc = sign_args(e, what, N, msg, msg_off, pre, pre_off, sig_at);
    if (rc < 0) return rc;
    CK(cudaSetDevice(e->device));
    std::vector<int> set(N);
    std::vector<int32_t> creator(N);
    for (int v = 0; v < B; v++)
        for (int r = offsets[v]; r < offsets[v + 1]; r++) { set[r] = v; creator[r] = engines[v]->sign_member; }
    rc = sign_run(e, N, set.data(), engines, B, msg, msg_off, pre, pre_off, sig_at, sig_out, ids_out);
    if (rc < 0) return rc;
    if (!index_out) return SW_OK;
    return ingest_views(engines, B, offsets, ids_out, p0_ids, p1_ids, creator.data(), t, sig_out, nullptr, index_out, count_out);
}

int sw_lookup(sw_engine *e, int n, const uint8_t *ids, int32_t *index_out) {
    if (!e || n < 0 || (n > 0 && (!ids || !index_out))) return fail(e, SW_E_ARG, "bad argument");
    for (int i = 0; i < n; i++) {
        Id32 k;
        memcpy(k.data(), ids + (size_t)32 * i, 32);
        auto it = e->ids.find(k);
        index_out[i] = it == e->ids.end() ? -1 : it->second;
    }
    return SW_OK;
}

int sw_get_ids(sw_engine *e, int first, int n, uint8_t *out) {
    if (!e || first < 0 || n < 0 || (n > 0 && !out)) return fail(e, SW_E_ARG, "bad argument");
    if ((i64)first + n > e->n_events) return fail(e, SW_E_KEY, "sw_get_ids: [%d,%d) out of range", first, first + n);
    for (int i = 0; i < n; i++) {
        const size_t x = (size_t)first + i;
        if (x < e->id_of.size()) memcpy(out + (size_t)32 * i, e->id_of[x].data(), 32);
        else memset(out + (size_t)32 * i, 0, 32);
    }
    return SW_OK;
}

// ---- sync: the sending end of Node.sync (swirld.py:125-126, 154-161, utils.py:24-34), selected on the GPU
namespace {
// The refusals the sync calls share: view v's head must be divided (its can_see row is complete), and its summary
// entries heights or -1
int sync_args(sw_engine *e, const sw_engine *x, int v, int head, const int32_t *summary, const char *what) {
    if (head < 0 || head >= x->n_divided)
        return fail(e, SW_E_ARG, "%s: view %d: head %d is not a divided event (%d divided)", what, v, head, x->n_divided);
    for (int c = 0; summary && c < x->M; c++)
        if (summary[c] < -1) return fail(e, SW_E_ARG, "%s: view %d: summary[%d] = %d < -1", what, v, c, summary[c]);
    return 0;
}

SyncParams sync_params(const sw_engine *x, int head) {
    SyncParams P{};
    P.row = x->d_row.get(); P.height = x->d_height.get(); P.creator = x->d_creator.get(); P.p0 = x->d_p0.get(); P.p1 = x->d_p1.get();
    P.t = x->d_t.get(); P.sig = x->d_sig.get(); P.M = x->M; P.head = head;
    return P;
}

// The kernels of a sync call run on the stream of `e`, the first view's, after the copies each view has appended (the
// rows of its divided events are written there or on its compute stream): what sw_get_can_see waits for.  No view
// waits for or gives up a round-stream piece, which writes rounds only.
int sync_enter(sw_engine *e, sw_engine *const *views, int B) {
    for (int v = 0; v < B; v++)
        if (wait_appends(views[v], -1) < 0) { e->err = views[v]->err; return SW_E_CUDA; }
    return views_enter(e, views, B);
}

extern "C++" template <class T> T *sec(char *base, size_t off) { return reinterpret_cast<T *>(base + off); }

// The summaries of B views (heads[v] divided, checked) into out, concatenated by view: one launch, one synchronisation.
// `batch`: the parameters go over as the device array of the views (the batched instance), else by value (B = 1).
int sync_summary(sw_engine *e, sw_engine *const *views, int B, const int *heads, int32_t *out, bool batch) {
    size_t MT = 0;
    for (int v = 0; v < B; v++) MT += views[v]->M;
    const size_t in_bytes = align256(sizeof(SyncParams) * B), out_bytes = sizeof(int32_t) * MT;
    if (grow(e, in_bytes, e->d_sync.cap(), sized(e->d_sync, std::max(in_bytes, 2 * e->d_sync.cap())),
             sized(e->h_sync_in, std::max(in_bytes, 2 * e->d_sync.cap()))) < 0 ||
        grow(e, out_bytes, e->h_sync_out.cap(), sized(e->h_sync_out, std::max(out_bytes, 2 * e->h_sync_out.cap()))) < 0)
        return SW_E_CUDA;
    if (sync_enter(e, views, B) < 0) return SW_E_CUDA;
    int32_t *hout = sec<int32_t>(e->h_sync_out.get(), 0);
    SyncParams *Pv = sec<SyncParams>(e->h_sync_in.get(), 0);
    for (int v = 0, o = 0; v < B; o += views[v]->M, v++) {
        Pv[v] = sync_params(views[v], heads[v]);
        Pv[v].heights_out = hout + o;
    }
    cudaStream_t st = e->stream.get();
    if (batch) {
        CK(cudaMemcpyAsync(e->d_sync.get(), Pv, sizeof(SyncParams) * B, cudaMemcpyHostToDevice, st));
        k_sync_summary<<<dim3(1, B), SY_THREADS, 0, st>>>((const SyncParams *)e->d_sync.get());
        e->stats.h2d_bytes += sizeof(SyncParams) * B;
    } else {
        k_sync_summary<<<1, SY_THREADS, 0, st>>>(Pv[0]);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    memcpy(out, hout, out_bytes);
    e->stats.kernel_launches += 1;
    e->stats.d2h_bytes += out_bytes;
    return SW_OK;
}

// Where a sync reply's columns sit in the output block, for `rows` rows
struct ReplyLayout {
    size_t hdr, index, creator, p0, p1, t, sig, bytes;
    ReplyLayout(int B, size_t rows) {
        hdr = 0; index = align256(sizeof(int32_t) * (2 * B + 2)); creator = index + align256(4 * rows);
        p0 = creator + align256(4 * rows); p1 = p0 + align256(4 * rows); t = p1 + align256(4 * rows);
        sig = t + align256(8 * rows); bytes = sig + 64 * rows;
    }
};

// A view's reply rows and the rows' ids, copied out of the output block: `j` rows from block row `at` to caller row
// `to`.  The id columns need an id for every selected event and every parent it names.
struct ReplyOut {
    int32_t *index; uint8_t *ids, *p0_ids, *p1_ids; int32_t *creator; double *t; uint8_t *sig;
};

int reply_ids_ok(sw_engine *e, const sw_engine *x, int v, const ReplyLayout &L, char *blk, int at, int n, const ReplyOut &O,
                 const char *what) {
    const Id32 zero{};
    auto has = [&](int i) { return i < 0 || ((size_t)i < x->id_of.size() && x->id_of[i] != zero); };
    for (int j = at; j < at + n; j++) {
        const int i = sec<int32_t>(blk, L.index)[j];
        if ((O.ids && !has(i)) || (O.p0_ids && !has(sec<int32_t>(blk, L.p0)[j])) || (O.p1_ids && !has(sec<int32_t>(blk, L.p1)[j])))
            return fail(e, SW_E_ARG, "%s: view %d: event %d of the reply (or a parent) has no id (it came through sw_append)", what, v, i);
    }
    return 0;
}

void reply_copy(const sw_engine *x, const ReplyLayout &L, char *blk, int at, int n, const ReplyOut &O) {
    const int32_t *ix = sec<int32_t>(blk, L.index) + at, *p0 = sec<int32_t>(blk, L.p0) + at, *p1 = sec<int32_t>(blk, L.p1) + at;
    if (O.index) memcpy(O.index + at, ix, 4 * (size_t)n);
    if (O.creator) memcpy(O.creator + at, sec<int32_t>(blk, L.creator) + at, 4 * (size_t)n);
    if (O.t) memcpy(O.t + at, sec<double>(blk, L.t) + at, 8 * (size_t)n);
    if (O.sig) memcpy(O.sig + (size_t)64 * at, sec<uint8_t>(blk, L.sig) + (size_t)64 * at, (size_t)64 * n);
    auto put = [&](uint8_t *dst, const int32_t *src) {
        if (!dst) return;
        for (int j = 0; j < n; j++) {
            if (src[j] < 0) memset(dst + (size_t)32 * (at + j), 0, 32);
            else memcpy(dst + (size_t)32 * (at + j), x->id_of[src[j]].data(), 32);
        }
    };
    put(O.ids, ix); put(O.p0_ids, p0); put(O.p1_ids, p1);
}

// The replies of B views (arguments checked) to the summaries, concatenated by view: count, scan and select in three
// launches on the first view's stream, one synchronisation.  counts_out[v] / offsets_out[0..B] are written when the
// call succeeds; on SW_E_CAPACITY (the replies hold more than `cap` rows) only counts_out is.
int sync_reply(sw_engine *e, sw_engine *const *views, int B, const int *heads, const int32_t *summaries, int cap,
               int32_t *counts_out, int32_t *offsets_out, const ReplyOut &O, bool batch, const char *what) {
    // tiles of [0, head] per view, and the most rows the replies can hold
    std::vector<int32_t> tile0(B + 1, 0);
    size_t MT = 0, bound = 0;
    int maxtiles = 0, maxM = 0;
    for (int v = 0; v < B; v++) {
        const int nt = (heads[v] + SY_TILE) / SY_TILE;
        tile0[v + 1] = tile0[v] + nt;
        maxtiles = std::max(maxtiles, nt);
        maxM = std::max(maxM, views[v]->M);
        MT += views[v]->M;
        bound += (size_t)heads[v] + 1;
    }
    const int T = tile0[B];
    const size_t rows = std::min<size_t>((size_t)std::max(cap, 0), bound);
    // the input block: parameters | tile starts | summaries, then the device-only scratch: tile counts | offsets | fits
    const size_t o_t0 = align256(sizeof(SyncParams) * B), o_sum = o_t0 + align256(sizeof(int32_t) * (B + 1));
    const size_t in_bytes = o_sum + align256(sizeof(int32_t) * MT);
    const size_t o_cnt = in_bytes, o_off = o_cnt + align256(sizeof(int32_t) * T), o_fits = o_off + align256(sizeof(int32_t) * (T + 1));
    const size_t dev_bytes = o_fits + 256;
    const ReplyLayout L(B, rows);
    if (grow(e, dev_bytes, e->d_sync.cap(), sized(e->d_sync, std::max(dev_bytes, 2 * e->d_sync.cap())),
             sized(e->h_sync_in, std::max(dev_bytes, 2 * e->d_sync.cap()))) < 0 ||
        grow(e, L.bytes, e->h_sync_out.cap(), sized(e->h_sync_out, std::max(L.bytes, 2 * e->h_sync_out.cap()))) < 0)
        return SW_E_CUDA;
    if (sync_enter(e, views, B) < 0) return SW_E_CUDA;
    char *hin = e->h_sync_in.get(), *din = e->d_sync.get(), *blk = e->h_sync_out.get();
    SyncParams *Pv = sec<SyncParams>(hin, 0);
    memcpy(hin + o_t0, tile0.data(), sizeof(int32_t) * (B + 1));
    memcpy(hin + o_sum, summaries, sizeof(int32_t) * MT);
    for (int v = 0, m = 0; v < B; m += views[v]->M, v++) {
        SyncParams &P = Pv[v];
        P = sync_params(views[v], heads[v]);
        P.summary = sec<int32_t>(din, o_sum) + m;
        P.tile_cnt = sec<int32_t>(din, o_cnt); P.tile_off = sec<int32_t>(din, o_off); P.fits = sec<int32_t>(din, o_fits);
        P.o_index = sec<int32_t>(blk, L.index); P.o_creator = sec<int32_t>(blk, L.creator);
        P.o_p0 = sec<int32_t>(blk, L.p0); P.o_p1 = sec<int32_t>(blk, L.p1); P.o_t = sec<double>(blk, L.t); P.o_sig = sec<uint8_t>(blk, L.sig);
        P.tile0 = tile0[v]; P.ntiles = tile0[v + 1] - tile0[v];
    }
    cudaStream_t st = e->stream.get();
    const size_t copy = in_bytes;
    CK(cudaMemcpyAsync(din, hin, copy, cudaMemcpyHostToDevice, st));
    const size_t smem = sizeof(int) * 2 * maxM;
    int32_t *hdr = sec<int32_t>(blk, L.hdr);
    if (batch) {
        const SyncParams *dP = (const SyncParams *)din;
        k_sync_count<<<dim3(maxtiles, B), SY_THREADS, smem, st>>>(dP);
        k_sync_scan<<<1, 1024, 0, st>>>(sec<int32_t>(din, o_cnt), T, sec<int32_t>(din, o_t0), B, (int)rows,
                                         sec<int32_t>(din, o_off), sec<int32_t>(din, o_fits), hdr);
        k_sync_select<<<dim3(maxtiles, B), SY_THREADS, smem, st>>>(dP);
    } else {
        k_sync_count<<<maxtiles, SY_THREADS, smem, st>>>(Pv[0]);
        k_sync_scan<<<1, 1024, 0, st>>>(sec<int32_t>(din, o_cnt), T, sec<int32_t>(din, o_t0), B, (int)rows,
                                         sec<int32_t>(din, o_off), sec<int32_t>(din, o_fits), hdr);
        k_sync_select<<<maxtiles, SY_THREADS, smem, st>>>(Pv[0]);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    e->stats.kernel_launches += 3;
    e->stats.h2d_bytes += (i64)copy;
    const int total = hdr[0];
    e->stats.d2h_bytes += (i64)sizeof(int32_t) * (2 * B + 2) + (total <= (i64)rows ? (i64)total * (4 * 5 + 8 + 64) : 0);
    if ((size_t)total > rows || total > cap) {
        memcpy(counts_out, hdr + 1, sizeof(int32_t) * B);
        return fail(e, SW_E_CAPACITY, "%s: the reply holds %d events, cap is %d", what, total, cap);
    }
    for (int v = 0; v < B; v++)
        if (reply_ids_ok(e, views[v], v, L, blk, hdr[1 + B + v], hdr[1 + v], O, what) < 0) return SW_E_ARG;
    for (int v = 0; v < B; v++) reply_copy(views[v], L, blk, hdr[1 + B + v], hdr[1 + v], O);
    memcpy(counts_out, hdr + 1, sizeof(int32_t) * B);
    if (offsets_out) memcpy(offsets_out, hdr + 1 + B, sizeof(int32_t) * (B + 1));
    return SW_OK;
}

// the checks of the batched calls: views, then every head and summary, before anything runs
int sync_batch_args(sw_engine *const *engines, int B, const int *heads, const int32_t *summaries, const char *what) {
    int rc = check_views(engines, B, what, false, false);
    if (rc < 0) return rc;
    sw_engine *e = engines[0];
    for (int v = 0, m = 0; v < B; m += engines[v]->M, v++)
        if (sync_args(e, engines[v], v, heads[v], summaries ? summaries + m : nullptr, what) < 0) return SW_E_ARG;
    return 0;
}
}  // namespace

int sw_sync_summary(sw_engine *e, int head, int32_t *heights_out) {
    if (!e || !heights_out) return fail(e, SW_E_ARG, "bad argument");
    if (e->nranks > 1) return fail(e, SW_E_UNSUPPORTED, "sw_sync_summary: one rank of a multi-GPU engine");
    if (sync_args(e, e, 0, head, nullptr, "sw_sync_summary") < 0) return SW_E_ARG;
    CK(cudaSetDevice(e->device));
    sw_engine *views[1] = {e};
    return sync_summary(e, views, 1, &head, heights_out, false);
}

int sw_batch_sync_summary(sw_engine *const *engines, int B, const int *heads, int32_t *out) {
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    if (!e || !heads || !out) return fail(e, SW_E_ARG, "bad argument");
    int rc = sync_batch_args(engines, B, heads, nullptr, "sw_batch_sync_summary");
    if (rc < 0) return rc;
    CK(cudaSetDevice(e->device));
    return sync_summary(e, engines, B, heads, out, true);
}

int sw_sync_reply(sw_engine *e, int head, const int32_t *summary, int cap, int32_t *index_out, int32_t *count_out,
                  uint8_t *ids, uint8_t *p0_ids, uint8_t *p1_ids, int32_t *creator, double *t, uint8_t *sig) {
    const char *what = "sw_sync_reply";
    if (!e || !summary || !count_out || cap < 0 || (cap > 0 && !index_out)) return fail(e, SW_E_ARG, "bad argument");
    if (e->nranks > 1) return fail(e, SW_E_UNSUPPORTED, "%s: one rank of a multi-GPU engine", what);
    if (sync_args(e, e, 0, head, summary, what) < 0) return SW_E_ARG;
    CK(cudaSetDevice(e->device));
    sw_engine *views[1] = {e};
    int32_t cnt = 0;
    const int rc = sync_reply(e, views, 1, &head, summary, cap, &cnt, nullptr, ReplyOut{index_out, ids, p0_ids, p1_ids, creator, t, sig}, false, what);
    if (rc == SW_OK || rc == SW_E_CAPACITY) *count_out = cnt;
    return rc < 0 ? rc : cnt;
}

int sw_batch_sync_reply(sw_engine *const *engines, int B, const int *heads, const int32_t *summaries, int cap,
                        int32_t *offsets_out, int32_t *counts_out, int32_t *index_out, uint8_t *ids, uint8_t *p0_ids,
                        uint8_t *p1_ids, int32_t *creator, double *t, uint8_t *sig) {
    const char *what = "sw_batch_sync_reply";
    sw_engine *e = (engines && B > 0) ? engines[0] : nullptr;
    if (!e || !heads || !summaries || !offsets_out || !counts_out || cap < 0 || (cap > 0 && !index_out))
        return fail(e, SW_E_ARG, "bad argument");
    int rc = sync_batch_args(engines, B, heads, summaries, what);
    if (rc < 0) return rc;
    CK(cudaSetDevice(e->device));
    std::vector<int32_t> cnt(B);
    rc = sync_reply(e, engines, B, heads, summaries, cap, cnt.data(), offsets_out, ReplyOut{index_out, ids, p0_ids, p1_ids, creator, t, sig}, true, what);
    if (rc == SW_OK || rc == SW_E_CAPACITY) memcpy(counts_out, cnt.data(), sizeof(int32_t) * B);
    return rc;
}

// ---- checkpoint / resume: the engine's whole state as one binary file (sections of SoA columns)
namespace {
struct CkptHeader {
    char magic[8];
    int32_t version, M, cap, C, Rcap, wide, NJ, n_events, n_divided, n_tx, n_rowed, rounds;
    uint32_t rb_epoch, n_ids;
};
const char CKPT_MAGIC[8] = {'S', 'W', 'B', '2', 'C', 'K', 'P', 'T'};

bool put_host(FILE *f, const void *p, size_t bytes) {
    uint64_t nb = bytes;
    return fwrite(&nb, 8, 1, f) == 1 && (bytes == 0 || fwrite(p, 1, bytes, f) == bytes);
}
bool put_dev(sw_engine *e, FILE *f, const void *d, size_t bytes, std::vector<char> &tmp) {
    uint64_t nb = bytes;
    if (fwrite(&nb, 8, 1, f) != 1) return false;
    const size_t CH = (size_t)64 << 20;
    for (size_t o = 0; o < bytes; o += CH) {
        const size_t k = std::min(CH, bytes - o);
        tmp.resize(k);
        if (cudaMemcpyAsync(tmp.data(), (const char *)d + o, k, cudaMemcpyDeviceToHost, e->stream.get()) != cudaSuccess) return false;
        if (cudaStreamSynchronize(e->stream.get()) != cudaSuccess) return false;
        if (fwrite(tmp.data(), 1, k, f) != k) return false;
    }
    return true;
}
bool get_host(FILE *f, void *p, size_t bytes) {
    uint64_t nb = 0;
    return fread(&nb, 8, 1, f) == 1 && nb == bytes && (bytes == 0 || fread(p, 1, bytes, f) == bytes);
}
bool get_dev(sw_engine *e, FILE *f, void *d, size_t bytes, std::vector<char> &tmp) {
    uint64_t nb = 0;
    if (fread(&nb, 8, 1, f) != 1 || nb != bytes) return false;
    const size_t CH = (size_t)64 << 20;
    for (size_t o = 0; o < bytes; o += CH) {
        const size_t k = std::min(CH, bytes - o);
        tmp.resize(k);
        if (fread(tmp.data(), 1, k, f) != k) return false;
        if (cudaMemcpyAsync((char *)d + o, tmp.data(), k, cudaMemcpyHostToDevice, e->stream.get()) != cudaSuccess) return false;
        if (cudaStreamSynchronize(e->stream.get()) != cudaSuccess) return false;
    }
    return true;
}

// The file: the header, the stake (sw_load needs it to create the engine), then these sections in this order, each
// sized from the header's counts.  `idrec`: the id records, 36 bytes each (32-byte id, arrival index).  Version 2 adds
// the consensus times and rounds received of the ordered positions behind them.
constexpr int32_t CKPT_VERSION = 2;
struct Section { void *p; size_t bytes; bool dev; };
std::vector<Section> ckpt_sections(sw_engine *e, const CkptHeader &H, std::vector<uint8_t> &idrec) {
    const size_t M = H.M, n = H.n_events, nd = H.n_divided, nr = H.n_rowed, NJ = H.NJ, R = H.rounds, RM = R * M;
    const size_t i4 = sizeof(int32_t), ntx = H.n_tx;
    const Section SM = H.wide ? Section{e->d_SMw.get(), sizeof(unsigned) * nd * NJ, true} : Section{e->d_SM.get(), sizeof(u64) * nd, true};
    const Section S = H.wide ? Section{e->d_Sw.get(), sizeof(unsigned) * RM * NJ, true} : Section{e->d_S.get(), sizeof(u64) * RM, true};
    std::vector<Section> v = {
        {e->h_creator.data(), i4 * n, false}, {e->h_head.data(), i4 * M, false}, {e->h_count.data(), i4 * M, false},
        {e->h_height.get(), i4 * n, false}, {e->h_seq.get(), i4 * n, false}, {e->h_stale.get(), n, false},
        {e->d_p0.get(), i4 * n, true}, {e->d_p1.get(), i4 * n, true}, {e->d_creator.get(), i4 * n, true}, {e->d_t.get(), sizeof(double) * n, true},
        {e->d_sig.get(), 64 * n, true}, {e->d_row.get(), i4 * nr * M, true}, {e->d_round.get(), i4 * nd, true}, {e->d_wit.get(), nd, true},
        SM, {e->d_famous_ev.get(), n, true}, {e->d_idx.get(), i4 * n, true}, {e->d_tx.get(), i4 * (size_t)H.n_tx, true},
        {e->d_W.get(), i4 * RM, true}, {e->d_Wf.get(), i4 * RM, true}, {e->d_famous.get(), RM, true}, {e->d_coin.get(), RM, true},
        S, {e->d_consensus.get(), R, true}, {e->d_lastord.get(), i4 * M, true}, {e->d_cs_carry.get(), i4 * M, true}, {e->d_rbtot.get(), i4 * M, true},
        {e->d_gchain.get(), i4 * M * RB_RING, true}, {e->d_scal.get(), i4 * SC_COUNT, true}, {idrec.data(), idrec.size(), false}};
    if (H.version >= 2) { v.push_back({e->d_tx_ts, sizeof(double) * ntx, true}); v.push_back({e->d_tx_rr, i4 * ntx, true}); }
    return v;
}
}  // namespace

int sw_save(sw_engine *e, const char *path) {
    if (!e || !path) return fail(e, SW_E_ARG, "bad argument");
    if (e->nranks > 1) return fail(e, SW_E_UNSUPPORTED, "sw_save: checkpoint one rank of a multi-GPU engine is not supported");
    int rc = sw_sync(e);
    if (rc < 0) return rc;
    FILE *f = fopen(path, "wb");
    if (!f) return fail(e, SW_E_ARG, "sw_save: cannot open %s", path);
    const int M = e->M, n = e->n_events, nd = e->n_divided, nr = e->n_rowed;
    const int R = std::min(e->Rcap, e->h_scal.get()[SC_MAX_ROUND] + 2);
    CkptHeader H{};
    memcpy(H.magic, CKPT_MAGIC, 8);
    H.version = CKPT_VERSION; H.M = M; H.cap = e->cap; H.C = e->C; H.Rcap = e->Rcap; H.wide = e->wide ? 1 : 0; H.NJ = e->NJ;
    H.n_events = n; H.n_divided = nd; H.n_tx = e->n_tx; H.n_rowed = nr; H.rounds = R; H.rb_epoch = e->rb_epoch;
    H.n_ids = (uint32_t)e->ids.size();
    std::vector<uint8_t> idrec((size_t)36 * e->ids.size());
    { size_t o = 0; for (auto &kv : e->ids) { memcpy(&idrec[o], kv.first.data(), 32); memcpy(&idrec[o + 32], &kv.second, 4); o += 36; } }
    std::vector<char> tmp;
    bool ok = fwrite(&H, sizeof H, 1, f) == 1 && put_host(f, e->h_stake.data(), sizeof(i64) * M);
    for (const Section &s : ckpt_sections(e, H, idrec))
        ok = ok && (s.dev ? put_dev(e, f, s.p, s.bytes, tmp) : put_host(f, s.p, s.bytes));
    ok = (fclose(f) == 0) && ok;
    if (!ok) return fail(e, SW_E_ARG, "sw_save: write to %s failed", path);
    return SW_OK;
}

int sw_load(const char *path, int device, int capacity_events, sw_engine **out) {
    sw_engine *e = nullptr;
    if (!path || !out) return fail(e, SW_E_ARG, "bad argument");
    *out = nullptr;
    FILE *f = fopen(path, "rb");
    if (!f) return fail(e, SW_E_ARG, "sw_load: cannot open %s", path);
    CkptHeader H{};
    if (fread(&H, sizeof H, 1, f) != 1 || memcmp(H.magic, CKPT_MAGIC, 8) != 0 || H.version < 1 || H.version > CKPT_VERSION || H.M < 1 || H.M > SW_MAX_MEMBERS
        || (H.M > 64 && !H.wide)) {
        fclose(f);
        return fail(e, SW_E_ARG, "sw_load: %s is not a swirld_b200 checkpoint", path);
    }
    std::vector<i64> stake(H.M);
    if (!get_host(f, stake.data(), sizeof(i64) * H.M)) { fclose(f); return fail(e, SW_E_ARG, "sw_load: truncated file"); }
    const int cap = std::max(capacity_events > 0 ? capacity_events : H.cap, H.n_events);
    // the saved engine's kernel family, whatever SW_FORCE_WIDE says now
    int rc = create(H.M, cap, reinterpret_cast<const int64_t *>(stake.data()), H.C, device, H.wide != 0, &e);
    if (rc < 0) { fclose(f); return rc; }
    const int M = H.M, n = H.n_events, nd = H.n_divided, nr = H.n_rowed, R = H.rounds;
    if (R > e->Rcap || (int)e->wide != H.wide || e->NJ != H.NJ) { fclose(f); sw_destroy(e); return fail(nullptr, SW_E_ARG, "sw_load: checkpoint does not fit the engine"); }
    std::vector<char> tmp;
    std::vector<uint8_t> idrec((size_t)36 * H.n_ids);
    e->h_creator.resize(n);
    bool ok = true;
    for (const Section &s : ckpt_sections(e, H, idrec))
        ok = ok && (s.dev ? get_dev(e, f, s.p, s.bytes, tmp) : get_host(f, s.p, s.bytes));
    e->id_of.assign(n, Id32{});
    for (size_t o = 0; ok && o < idrec.size(); o += 36) {
        Id32 k; int32_t v; memcpy(k.data(), &idrec[o], 32); memcpy(&v, &idrec[o + 32], 4);
        e->ids.emplace(k, v);
        if (v >= 0 && v < n) e->id_of[v] = k;
    }
    fclose(f);
    if (!ok) { sw_destroy(e); return fail(nullptr, SW_E_ARG, "sw_load: %s is truncated or does not match its header", path); }
    // the derived columns live on the device too
    bool ok2 = cudaMemcpy(e->d_seq.get(), e->h_seq.get(), sizeof(int32_t) * n, cudaMemcpyHostToDevice) == cudaSuccess
        && cudaMemcpy(e->d_height.get(), e->h_height.get(), sizeof(int32_t) * n, cudaMemcpyHostToDevice) == cudaSuccess
        && cudaMemcpy(e->d_stale.get(), e->h_stale.get(), (size_t)n, cudaMemcpyHostToDevice) == cudaSuccess;
    // a version-1 file has no times or rounds received for what it had ordered: NaN (all bits set) and -1
    if (ok2 && H.version < 2)
        ok2 = cudaMemsetAsync(e->d_tx_ts, 0xff, sizeof(double) * (size_t)H.n_tx, e->stream.get()) == cudaSuccess
            && cudaMemsetAsync(e->d_tx_rr, 0xff, sizeof(int32_t) * (size_t)H.n_tx, e->stream.get()) == cudaSuccess
            && cudaStreamSynchronize(e->stream.get()) == cudaSuccess;
    if (!ok2) { sw_destroy(e); return fail(nullptr, SW_E_CUDA, "sw_load: device copy failed"); }
    e->n_events = n; e->n_divided = nd; e->n_tx = H.n_tx; e->n_rowed = nr; e->rb_epoch = H.rb_epoch;
    e->h_stale_cum.assign((size_t)n + 1, 0);
    for (int i = 0; i < n; i++) e->h_stale_cum[i + 1] = e->h_stale_cum[i] + e->h_stale.get()[i];
    std::vector<int32_t> cnt(M, 0);
    for (int i = 0; i < n; i++) {
        cnt[e->h_creator[i]]++;
        if ((i + 1) % sw_engine::SNAP == 0 || i + 1 == n) push_snapshot(e, i + 1, cnt);
    }
    e->stats.events = n; e->stats.events_divided = nd;
    *out = e;
    return SW_OK;
}

// ---- several GPUs of one box: exchange buffers over NVLink peer memory (CUDA IPC, one process per GPU)
int sw_peer_handle(sw_engine *e, void *handle_out64) {
    if (!e || !handle_out64) return fail(e, SW_E_ARG, "bad argument");
    if (!e->wide) return fail(e, SW_E_UNSUPPORTED, "the M <= 64 path does not shard (replicas only): no peer exchange");
    CK(cudaSetDevice(e->device));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, e->d_xbuf.get()));
    memcpy(handle_out64, &h, 64);
    CK(cudaIpcGetMemHandle(&h, e->d_row.get()));
    memcpy(reinterpret_cast<char *>(handle_out64) + 64, &h, 64);
    return SW_OK;
}

int sw_peer_connect(sw_engine *e, int rank, int nranks, const void *handles) {
    if (!e || !handles || nranks < 1 || nranks > 8 || rank < 0 || rank >= nranks) return fail(e, SW_E_ARG, "bad argument");
    if (!e->wide) return fail(e, SW_E_UNSUPPORTED, "the M <= 64 path does not shard (replicas only): no peer exchange");
    if (e->n_divided > 0) return fail(e, SW_E_ARG, "sw_peer_connect: connect before the first divide_rounds");
    CK(cudaSetDevice(e->device));
    for (int p = 0; p < nranks; p++) {
        if (p == rank) { e->x_peer[p] = e->d_xbuf.get(); e->row_peer[p] = e->d_row.get(); continue; }
        const char *hp = reinterpret_cast<const char *>(handles) + (size_t)SW_PEER_HANDLE_BYTES * p;
        CK(e->x_map[p].open(hp));
        e->x_peer[p] = e->x_map[p].get();
        CK(e->row_map[p].open(hp + 64));
        e->row_peer[p] = static_cast<int32_t *>(e->row_map[p].get());
    }
    // the ranks' barrier flag rows (128 bytes into the exchange buffer) as a device array
    unsigned *fl[8] = {nullptr};
    for (int p = 0; p < nranks; p++) fl[p] = reinterpret_cast<unsigned *>(reinterpret_cast<char *>(e->x_peer[p]) + 128);
    if (!e->d_xflags2.get()) CK(e->d_xflags2.alloc(8));
    CK(cudaMemcpy(e->d_xflags2.get(), fl, sizeof fl, cudaMemcpyHostToDevice));
    e->rank = rank; e->nranks = nranks;
    return SW_OK;
}

}  // extern "C"
