/*
 * swirld_b200.h -- C ABI of libswirld_b200.so, the H100 (sm_90a) engine for
 * py-swirld's consensus hot path.
 *
 * The reference (Lapin0t/py-swirld) has no FFI: its "operator interface" for this
 * path is the method surface of `swirld.Node` (swirld.py).  Each
 * entry point below replaces one of those methods / attributes; the Python class
 * `swirld_b200.node.GpuNode` binds them with ctypes and presents the reference's
 * own names (see INTEGRATION.md).  Index space: an event is its arrival index at
 * this node-view (int32, topological), a member is 0..M-1.
 *
 * Conventions: plain pointers and sizes only; every pointer argument is HOST
 * memory owned by the caller; device memory is owned by the engine; one CUDA
 * stream per engine; one caller thread per engine (the reference is single
 * threaded: README.md:27-28).  Functions return >= 0 on success and a negative
 * SW_E_* code on failure; sw_last_error() gives the text.  There is NO CPU
 * fallback: without a CUDA device sw_create fails with SW_E_CUDA.
 */
#ifndef SWIRLD_B200_H
#define SWIRLD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SW_OK            0
#define SW_E_ARG        -1   /* bad argument */
#define SW_E_INDEX      -2   /* reference would raise IndexError (swirld.py:305, one seer) */
#define SW_E_KEY        -3   /* reference would raise KeyError (unknown event / round) */
#define SW_E_CUDA       -4   /* CUDA runtime error or no device */
#define SW_E_CAPACITY   -5   /* capacity_events / round table exhausted */
#define SW_E_PARENT     -6   /* invalid parents: is_valid_event would be False (swirld.py:104-108) */
#define SW_E_FORK       -7   /* self-parent is not the creator's latest event (fork; swirld.py:110-112 TODO) */
#define SW_E_UNSUPPORTED -8  /* e.g. M above the compiled kernels' limit */

#define SW_MAX_MEMBERS  1024 /* member sets are ceil(M/32)-word masks; above 64 members the swirld_wide.cuh kernels run */

typedef struct sw_engine sw_engine;

/* Cumulative counters since sw_create / sw_reset (device times from CUDA events
 * recorded on the engine's stream around the kernels of each call). */
typedef struct sw_stats_t {
    double ms_divide_rounds;   /* every kernel of sw_divide_rounds (can_see scan, rounds, witnesses, k_strong) */
    double ms_decide_fame;     /* k_fame_* */
    double ms_find_order;      /* k_order_* */
    double ms_can_see;         /* subset of ms_divide_rounds spent in a stand-alone can_see kernel, 0 if fused */
    int64_t kernel_launches;   /* kernels of this library launched (a divide_rounds call whose rounds ran ahead on the
                                  round stream counts the launches the same call makes without it) */
    int64_t h2d_bytes;
    int64_t d2h_bytes;
    int64_t events;            /* events appended */
    int64_t events_divided;    /* events through divide_rounds */
    double ms_rounds_kernel;   /* subset of ms_divide_rounds spent in the round-number kernel itself
                                  (M <= 64: k_rb_prep + k_rounds_cluster + k_rounds_batch; above: k_rounds_wide);
                                  round kernels run ahead on the round stream (SW_ROUNDS_AHEAD) are not timed */
    int64_t rounds_cluster_launches;   /* launches of k_rounds_cluster (one view or several): 0 when the device cannot
                                          hold the 16-CTA cluster and every chunk ran on the grid-wide k_rounds_batch */
} sw_stats_t;

/* Node.__init__ state (swirld.py:38-72): M members, integer stake per member
 * (NULL = unit stake as in both reference drivers, swirld.py:334 / viz.py:36),
 * coin period C (swirld.py:17), room for capacity_events events.  SW_E_ARG for a
 * negative stake or a total above (2^63 - 1) / 3, whose triple overflows int64. */
int sw_create(int M, int capacity_events, const int64_t *stake, int coin_period,
              int device, sw_engine **out);
void sw_destroy(sw_engine *e);
/* Forget every event and all consensus state; keeps the allocations. */
int sw_reset(sw_engine *e);
/* Forget the consensus state (rounds, witnesses, fame, order) but keep the appended
 * event columns resident on the device: the next sw_divide_rounds starts at 0 again. */
int sw_rewind(sw_engine *e);
const char *sw_last_error(const sw_engine *e);   /* e may be NULL: last create error */

/* Node.add_event (swirld.py:114-120) for n events in arrival order, SoA columns:
 * p0/p1 = self/other parent index (-1,-1 for a root: ev.p == ()), creator,
 * t = Event.t (swirld.py:91), sig = Event.s, 64 bytes each (swirld.py:92).
 * Checks what is_valid_event checks on the graph shape (swirld.py:104-108) and
 * the fork-free contract; copies the columns to the device and, for a batch of 4096
 * events or more, starts their can_see rows (swirld.py:203-205, 220) right away.  Both run
 * on the engine's copy stream beside the kernels of earlier calls (a caller that appends a
 * chunk or two ahead of its sw_divide_rounds calls hides them completely): when the columns are in
 * page-locked host memory they must stay unchanged until the next synchronising call
 * (sw_decide_fame, sw_find_order, sw_sync, any sw_get_*); pageable memory is staged
 * before the call returns. */
int sw_append(sw_engine *e, int n, const int32_t *p0, const int32_t *p1,
              const int32_t *creator, const double *t, const uint8_t *sig);

/* Node.add_event for B independent node-views in one call (each node of the simulation receives the events of its
 * sync, swirld.py:319-324): view v appends rows offsets[v] .. offsets[v+1] of the concatenated columns (as sw_append).
 * The views may differ in M; they share one device.  The views of at most 64 events go over packed in ONE copy and are
 * scattered by ONE kernel on the first engine's copy stream (charged to the first engine): the caller's arrays are free
 * again when the call returns.  Larger views make the copies (and can_see scan) their sw_append makes, under its
 * page-locked memory contract.
 * Argument errors refuse the whole call before anything runs, leave rc_out unwritten and put the message in the first
 * engine's sw_last_error: B < 1, a NULL or repeated engine, views on different devices or peer-connected to other GPUs
 * (SW_E_UNSUPPORTED), offsets that are not monotone (SW_E_ARG).  A view whose events sw_append would refuse (SW_E_PARENT,
 * SW_E_FORK, SW_E_CAPACITY, SW_E_ARG for a creator out of range) appends nothing: rc_out[v] gets that code and the
 * message is in that view's sw_last_error; the other views append normally (rc_out[v] = SW_OK).  Returns SW_OK when
 * every view appended, else the first failing view's code. */
int sw_batch_append(sw_engine *const *engines, int B, const int *offsets, const int32_t *p0, const int32_t *p1,
                    const int32_t *creator, const double *t, const uint8_t *sig, int32_t *rc_out);

/* Node.divide_rounds(events) (swirld.py:187-222) for the topologically sorted
 * events [first, first+n): can_see rows, round numbers, witness registration.
 * `first` must equal the number of events already divided. Asynchronous. */
int sw_divide_rounds(sw_engine *e, int first, int n);

/* Node.divide_rounds for B independent node-views in one call (the simulation's M nodes each recompute consensus on
 * nearly the same graph, swirld.py:331-345 / viz.py:35-46): engines[v] divides its events [first[v], first[v]+n[v]).
 * The views share one member count, kernel family and device (as sw_batch_decide_fame), and each takes the path its
 * single call would take:
 *  - a call of at most 16 events whose can_see rows are not behind (the reference's cadence): every such view in ONE
 *    launch, one thread block per view, at any M; stakes and coin periods may differ.  Asynchronous, like
 *    sw_divide_rounds: each view's stream waits for the launch, and nothing synchronises the host.
 *  - the other calls (M <= 64 only, one stake shape among them): the views' round kernels advance side by side -- one
 *    thread-block cluster per view (chunks of >= 2048 events), then ONE cooperative launch, each view on its own group
 *    of CTAs, for what is left: the path is latency-bound, so this is what fills the GPU.
 * A batch whose chunk-path views break those rules is refused as a whole before anything runs (SW_E_UNSUPPORTED), as are
 * views that differ in M, kernel family or device, a NULL or repeated engine and a bad range (SW_E_ARG).  Timings and
 * launches are charged to the first engine.  Results per view are identical to B separate sw_divide_rounds calls. */
int sw_batch_divide_rounds(sw_engine *const *engines, int B, const int *first, const int *n);

/* Node.decide_fame() (swirld.py:224-277).  Writes the new consensus rounds
 * (ascending) to new_c_out[0..cap) and returns their count. */
int sw_decide_fame(sw_engine *e, int32_t *new_c_out, int cap);

/* Node.find_order(new_c) (swirld.py:280-311).  Returns the number of events
 * appended to the consensus order by this call (the caller owns the print of
 * swirld.py:310-311). */
int sw_find_order(sw_engine *e, const int32_t *new_c, int n);
/* sw_find_order, and also: the events this call appended to the order, in order, with their consensus time (ts[x],
 * swirld.py:305) and round received (the r of swirld.py:283), into ev_out / ts_out / rr_out[0 .. return value).  cap must
 * be >= sw_n_divided - sw_n_transactions (SW_E_ARG before anything runs otherwise).  The first 1024 events come back in
 * the copy sw_find_order makes; a call that orders more copies the rest in one more round trip.  On an error the
 * device finds (SW_E_INDEX, SW_E_KEY) the output is unspecified. */
int sw_find_order_out(sw_engine *e, const int32_t *new_c, int n,
                      int32_t *ev_out, double *ts_out, int32_t *rr_out, int cap);

/* Node.decide_fame() and Node.find_order(new_c) for B independent node-views in one call each (the simulation's nodes
 * each run the reference's whole main loop, swirld.py:325-328).  The views share one member count (any M up to
 * SW_MAX_MEMBERS), one kernel family (the M <= 64 kernels, or the any-M kernels that SW_FORCE_WIDE=1 selects) and one
 * device; stakes and coin periods may differ.  Every view's kernels run side by side in a fixed number of launches on
 * the first engine's stream, after what each view has queued on its own; one copy brings back the scalars of all views
 * and the call synchronises once.  Timings and launches are charged to the first engine.
 * Each view ends with exactly the state and results B single calls would have left it.
 * Argument errors refuse the whole call before anything runs, leave count_out unwritten and put the message in the
 * first engine's sw_last_error: B < 1, a NULL or repeated engine, a view peer-connected to other GPUs, views that
 * differ in device, M or kernel family (SW_E_UNSUPPORTED); for decide_fame a view with nothing divided (SW_E_ARG); for
 * find_order offsets that are not monotone (SW_E_ARG) or a round outside the view's round table (SW_E_KEY).
 * Errors the device finds belong to their view: count_out[v] gets the code sw_decide_fame / sw_find_order would
 * have returned (e.g. SW_E_INDEX, a single seer) and the message is in that view's sw_last_error; the other views
 * complete normally.  Returns SW_OK when every view succeeded, else the first failing view's code. */
/* new_c_out is B x cap: row v holds view v's new consensus rounds, ascending; count_out[v] = their count.  A view that
 * brings more than 1024 new rounds costs one more copy. */
int sw_batch_decide_fame(sw_engine *const *engines, int B, int32_t *new_c_out, int cap, int32_t *count_out);
/* View v's rounds are new_c[offsets[v] .. offsets[v+1]) (an empty range does nothing); count_out[v] = events appended
 * to view v's order. */
int sw_batch_find_order(sw_engine *const *engines, int B, const int32_t *new_c, const int *offsets, int32_t *count_out);
/* sw_batch_find_order, and also: view v's output (as sw_find_order_out's) is packed at out_offsets[v] .. out_offsets[v+1]
 * of ev_out / ts_out / rr_out (B+1 entries, written by the call; a failed view's range is empty); cap must be >= the sum
 * over the views of sw_n_divided - sw_n_transactions (SW_E_ARG before anything runs otherwise).  The same launches and
 * one copy back as sw_batch_find_order; views that order more than 1024 events add one more round trip in all. */
int sw_batch_find_order_out(sw_engine *const *engines, int B, const int32_t *new_c, const int *offsets,
                            int32_t *count_out, int32_t *ev_out, double *ts_out, int32_t *rr_out,
                            int *out_offsets, int cap);

/* ---- views of the Node attributes (swirld.py:48-72) ---- */
int sw_members(const sw_engine *e);           /* n (swirld.py:40) */
int sw_n_events(const sw_engine *e);          /* len(hg) */
int sw_n_divided(const sw_engine *e);         /* len(round) */
int sw_max_round(sw_engine *e);               /* max(witnesses), -1 if none */
int sw_n_transactions(const sw_engine *e);    /* len(transactions) */
int sw_get_round(sw_engine *e, int first, int n, int32_t *out);          /* round[h] */
int sw_get_witness_flags(sw_engine *e, int first, int n, uint8_t *out);  /* h in witnesses[round[h]].values() */
int sw_get_famous(sw_engine *e, int first, int n, int8_t *out);          /* famous.get(h): -1 absent, 0, 1 */
int sw_get_can_see(sw_engine *e, int first, int n, int32_t *out);        /* can_see[h] as n x M, -1 absent */
int sw_get_witness_table(sw_engine *e, int first_round, int n_rounds, int32_t *out); /* witnesses[r][c], -1 absent */
int sw_get_consensus(sw_engine *e, int32_t *out, int cap);               /* sorted(consensus) -> count */
int sw_get_transactions(sw_engine *e, int first, int n, int32_t *out);   /* transactions[first:first+n] */
/* by order position, parallel to sw_get_transactions: [first, first+n) within [0, sw_n_transactions) */
int sw_get_consensus_times(sw_engine *e, int first, int n, double *out);    /* ts[x] of transactions[i], swirld.py:305 */
int sw_get_rounds_received(sw_engine *e, int first, int n, int32_t *out);   /* the r of swirld.py:283 that ordered it */
int sw_get_idx(sw_engine *e, int first, int n, int32_t *out);            /* idx.get(h, -1) */
int sw_get_height(sw_engine *e, int first, int n, int32_t *out);         /* height[h] (swirld.py:68) */

int sw_sync(sw_engine *e);                     /* wait for the stream, fold timings into stats */
int sw_stats(sw_engine *e, sw_stats_t *out);   /* implies sw_sync */
/* Write >= bytes of device memory (evicts L2) on the engine's stream; for benchmarks. */
int sw_flush_l2(sw_engine *e, int64_t bytes);
/* CUDA events on the engine's stream, slots 0..15: record, and elapsed ms between two
 * recorded slots (synchronises on the later one). */
int sw_event_record(sw_engine *e, int slot);
int sw_event_elapsed_ms(sw_engine *e, int slot_a, int slot_b, double *ms_out);

/* Profiling aid: 16 cycle counters of the round kernels (tools/rounds_cycles.py). */
int sw_debug_counters(sw_engine *e, int64_t *out16, int clear);
/* Profiling aid: the cluster round kernel's per-CTA step log, kept only when the engine was created with the
 * environment variable SW_RC_STEPS = the number of steps to keep (tools/rc_steps.py; the record layout is in
 * swirld_rcluster.cuh).  Copies at most cap_words words (a 16-word header, then 16 words per step and CTA) and
 * returns the steps logged since the last clear (more than were kept if the log overflowed), 0 without a log. */
int sw_rc_step_log(sw_engine *e, uint32_t *out, int64_t cap_words, int clear);

/* ---- ingest: the step of Node.sync between the wire and divide_rounds (swirld.py:129-136, utils.py:8-21) in C++.
 * A batch of n events named by their 32-byte ids (BLAKE2b, swirld.py:95), parents given by id (32 zero bytes = none: a
 * root).  Ids the engine knows already are skipped; the others are put in a parents-first order (iterative DFS over the
 * batch; a cycle returns SW_E_ARG like toposort's ValueError), validated like sw_append validates (unknown parent,
 * parent shape, fork -- such an event, and whatever depends on it, is skipped: index -1), appended by ONE sw_append in
 * that order and entered in the engine's id -> index map.  index_out[i] = arrival index of input event i.  Returns
 * the number of events appended.  It checks no signature and no id: sw_ingest_verified does both on the GPU. */
int sw_ingest(sw_engine *e, int n, const uint8_t *ids, const uint8_t *p0_ids, const uint8_t *p1_ids,
              const int32_t *creator, const double *t, const uint8_t *sig, int32_t *index_out);

/* ---- is_valid_event's crypto (swirld.py:97-103) on the GPU: Ed25519 signatures with libsodium's verdicts, BLAKE2b ids.
 * The members' Ed25519 public keys, M x 32 bytes (member m = row m, the member order of the stake).  May be called
 * again to replace them.  A key libsodium would refuse (y not canonical, not on the curve, small order) is accepted
 * here and every signature under it then fails, as crypto_sign_verify_detached fails for it.  sw_reset and sw_rewind
 * keep the keys; they are not part of the checkpoint (an engine from sw_load has none until this is called). */
int sw_set_member_keys(sw_engine *e, const uint8_t *pk);

/* For n events: flags_out[i] bit 0 = sig[i] (64 bytes) is a valid Ed25519 signature by member creator[i] of
 * msg[msg_off[i] .. msg_off[i+1]) exactly when libsodium's crypto_sign_verify_detached (>= 1.0.18) accepts it; bit 1 =
 * BLAKE2b-256(pre[pre_off[i] .. pre_off[i+1])) == ids[i] (32 bytes).  Offsets are n+1 int64, monotone, starting at 0.
 * SW_E_ARG before anything runs, flags_out unwritten, for no keys, a creator out of range or bad offsets.  Runs on the
 * engine's stream (sw_event_record slots can bracket it); synchronous: returns SW_OK once flags_out is written. */
int sw_verify_events(sw_engine *e, int n, const int32_t *creator, const uint8_t *sig,
                     const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off,
                     const uint8_t *ids, uint8_t *flags_out);

/* sw_ingest, and also: every NEW event of the batch (an id the engine does not know yet, swirld.py:130) must pass
 * sw_verify_events with flags == 3, or it is skipped like an invalid event (index -1), and so is whatever depends on
 * it.  A known id is not checked again.  Only the new events go to the GPU, in one sw_verify_events pass.  SW_E_ARG
 * before anything runs for no keys or bad offsets (msg_off / pre_off as sw_verify_events, n+1 entries). */
int sw_ingest_verified(sw_engine *e, int n, const uint8_t *ids, const uint8_t *p0_ids, const uint8_t *p1_ids,
                       const int32_t *creator, const double *t, const uint8_t *sig,
                       const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off,
                       int32_t *index_out);
/* sw_ingest_verified for B independent node-views in one call (each node of the simulation ingests the reply of its
 * sync, swirld.py:129-136): view v ingests rows offsets[v] .. offsets[v+1] of the concatenated columns (as
 * sw_batch_append lays them out); msg_off / pre_off have offsets[B] + 1 entries over the whole concatenation, monotone
 * from 0, and index_out is laid out like the rows.  Each view ends with exactly the state, index_out and count its own
 * sw_ingest_verified of its rows would have given it.  The events the views would verify are verified ONCE per distinct
 * event: copies in several views share one verdict when their creator has the same 32-byte key in each view's key set
 * and their id, signature, message and preimage are byte-identical (a copy tampered under the same id is another event).
 * All of them go to the GPU in one copy and two kernels on the first engine's stream, with one synchronisation;
 * *n_verified_out (may be NULL) gets their number.  The accepted events append as sw_batch_append appends them.  The
 * views may differ in M and key sets; they share one device.  Launches and timings are charged to the first engine.
 * Argument errors refuse the whole call before anything runs, leave count_out unwritten and put the message in the
 * first engine's sw_last_error: B < 1, a NULL or repeated engine, views on different devices or peer-connected to other
 * GPUs (SW_E_UNSUPPORTED), a view with no member keys, bad row or byte offsets (SW_E_ARG).  A view's own failure (a
 * batch that is not a DAG, SW_E_ARG; capacity, SW_E_CAPACITY) changes nothing of that view: count_out[v] gets the code
 * and the message is in that view's sw_last_error; the other views ingest normally (count_out[v] = events appended).
 * Returns SW_OK when every view succeeded, else the first failing view's code. */
int sw_batch_ingest_verified(sw_engine *const *engines, int B, const int *offsets,
                             const uint8_t *ids, const uint8_t *p0_ids, const uint8_t *p1_ids,
                             const int32_t *creator, const double *t, const uint8_t *sig,
                             const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off,
                             int32_t *index_out, int32_t *count_out, int32_t *n_verified_out);
int sw_lookup(sw_engine *e, int n, const uint8_t *ids, int32_t *index_out);   /* id -> arrival index, -1 unknown */

/* ---- a node's own new events (Node.new_event, swirld.py:82-95, 139-144) on the GPU: Ed25519 signatures byte for byte
 * as libsodium's crypto_sign_detached makes them, BLAKE2b-256 ids, and the events entered into the view.
 * The view's signing key: sk is libsodium's 64-byte secret key (seed || pk).  Requires member keys
 * (sw_set_member_keys), and sk[32..64) must be member `member`'s key; the device then checks that [a]B encodes to it.
 * Otherwise SW_E_ARG, and the engine keeps the signing key it had (if any).  Only the expanded key (a, prefix) is kept,
 * in device memory; the staging copies of sk are wiped before the call returns.  Setting a key again replaces it.
 * sw_reset and sw_rewind keep it; sw_save never writes it (an engine from sw_load has none); sw_destroy overwrites it
 * on the device before freeing.  Signing is constant time in the key and the nonce. */
int sw_set_signing_key(sw_engine *e, int member, const uint8_t *sk);

/* n events by the view's signing member.  msg[msg_off[i] .. msg_off[i+1]) is event i's signed message,
 * dumps((d, p, t, pk)); pre[pre_off[i] .. pre_off[i+1]) is its preimage dumps(Event(d, p, t, pk, s)) with any 64 bytes
 * at sig_at[i] in place of s.  Offsets are n+1 int64, monotone from 0.  sig_out gets the 64-byte signatures and ids_out
 * the 32-byte ids, BLAKE2b-256 of the preimage with the signature in place.  With index_out NULL that is all (returns
 * SW_OK).  Else the events are also ingested exactly as sw_ingest ingests the rows (ids_out, p0_ids, p1_ids, creator =
 * the signing member, t, sig_out): parents by id, an unknown parent, a bad shape or a fork gives -1; returns the number
 * appended.  PRECONDITION: msg, pre, p0_ids, p1_ids and t describe the same event; the engine does not parse pickle.
 * SW_E_ARG before anything runs for no signing key, bad offsets or a sig_at outside [0, len - 64].  One pinned block
 * in, one launch on the engine's stream, one copy back, one synchronisation (then the ingest's own append). */
int sw_new_events(sw_engine *e, int n, const uint8_t *p0_ids, const uint8_t *p1_ids, const double *t,
                  const uint8_t *msg, const int64_t *msg_off, const uint8_t *pre, const int64_t *pre_off,
                  const int64_t *sig_at, uint8_t *sig_out, uint8_t *ids_out, int32_t *index_out);
/* sw_new_events for B node-views in one call: rows offsets[v] .. offsets[v+1] (offsets[0] = 0) belong to view v and are
 * signed by its key; msg_off / pre_off have offsets[B] + 1 entries over the whole concatenation and every other column
 * is laid out like the rows.  The views share one device and may differ in M.  Every row is signed in the same launch on
 * the first engine's stream; with index_out, the accepted rows append as sw_batch_ingest_verified's do and count_out[v]
 * gets view v's count.  Each view's outputs and state equal those of its own single call, byte for byte.  Argument
 * errors refuse the whole call before anything runs, as sw_batch_ingest_verified's do (a view without a signing key:
 * SW_E_ARG).  A view's own failure (capacity: SW_E_CAPACITY) goes to count_out[v] and that view's sw_last_error. */
int sw_batch_new_events(sw_engine *const *engines, int B, const int *offsets, const uint8_t *p0_ids,
                        const uint8_t *p1_ids, const double *t, const uint8_t *msg, const int64_t *msg_off,
                        const uint8_t *pre, const int64_t *pre_off, const int64_t *sig_at, uint8_t *sig_out,
                        uint8_t *ids_out, int32_t *index_out, int32_t *count_out);

/* Every event's 32-byte id from the engine's id map (sw_ingest), by arrival index, for [first, first+n) of the appended
 * events: 32 zero bytes for an event that has none (it came through sw_append).  SW_E_KEY for a range beyond them. */
int sw_get_ids(sw_engine *e, int first, int n, uint8_t *out);

/* ---- sync: the sending end of Node.sync (swirld.py:125-126, 154-161), selected on the GPU from the can_see table.
 * The requester's summary (swirld.py:125-126): heights_out[c] = height[can_see[head][c]], the height of the latest
 * event of member c that `head` sees, -1 where it sees none; M entries.  `head` must be divided (head < sw_n_divided),
 * else SW_E_ARG.  Synchronous; reads what pending appends and their can_see scans write, and neither waits for nor
 * gives up rounds computed ahead (SW_ROUNDS_AHEAD). */
int sw_sync_summary(sw_engine *e, int head, int32_t *heights_out);

/* The responder's reply to a summary (ask_sync, swirld.py:154-161, utils.py:24-34): the events a BFS from `head` over
 * the parents the requester lacks yields, which on a fork-free graph are
 *     {head} u { x < head : x <= can_see[head][creator x]  and  (summary[creator x] = -1  or  height[x] > summary[creator x]) }
 * in ascending arrival index (a topological order: sw_ingest takes the rows as they are).  `head` is in the reply even
 * when the requester has it.  PRECONDITION: summary (M entries) comes from a view of the same fork-free gossip, as
 * sw_sync_summary makes it; for an arbitrary summary the closed form can select events the BFS does not reach.
 * index_out[0..count) gets the events; each row pointer that is not NULL gets their columns in sw_ingest's layout:
 * ids / p0_ids / p1_ids 32 bytes each (from the id map; parents of a root are 32 zero bytes), creator, t, sig 64 bytes.
 * Returns the count, also in *count_out.  Errors, before anything is written: NULL engine, summary or count_out, cap < 0,
 * a head that is not divided or a summary entry < -1 (SW_E_ARG); an id column asked for while a selected event (or a
 * parent it names) has no id, i.e. came through sw_append (SW_E_ARG); a reply of more than `cap` events: only
 * *count_out is written, with the exact count (SW_E_CAPACITY).  Three launches and one synchronisation; stream
 * ordering as sw_sync_summary. */
int sw_sync_reply(sw_engine *e, int head, const int32_t *summary, int cap, int32_t *index_out, int32_t *count_out,
                  uint8_t *ids, uint8_t *p0_ids, uint8_t *p1_ids, int32_t *creator, double *t, uint8_t *sig);

/* sw_sync_summary and sw_sync_reply for B independent node-views in one call: view v answers with heads[v].  The views
 * share one device and may differ in M.  Summaries (in and out) are concatenated by view, M of that view each.  The
 * reply rows come out concatenated by view, view v's at offsets_out[v] .. offsets_out[v+1] (B+1 entries), exactly as
 * sw_batch_ingest_verified takes them, and counts_out[v] is view v's count; each view's rows equal its own single
 * call's byte for byte.  The same launches as one single call, on the first engine's stream, and one synchronisation.
 * Argument errors refuse the whole call before anything runs or is written (message in the first engine's
 * sw_last_error): B < 1, a NULL or repeated engine (SW_E_ARG), views on different devices or peer-connected to other
 * GPUs (SW_E_UNSUPPORTED), a head out of range or not divided, a summary entry < -1 (SW_E_ARG); for the reply also a
 * missing id as sw_sync_reply (SW_E_ARG).  A total above `cap` writes only counts_out, with exact counts, and returns
 * SW_E_CAPACITY. */
int sw_batch_sync_summary(sw_engine *const *engines, int B, const int *heads, int32_t *out);
int sw_batch_sync_reply(sw_engine *const *engines, int B, const int *heads, const int32_t *summaries, int cap,
                        int32_t *offsets_out, int32_t *counts_out, int32_t *index_out, uint8_t *ids, uint8_t *p0_ids,
                        uint8_t *p1_ids, int32_t *creator, double *t, uint8_t *sig);

/* ---- checkpoint / resume (the reference keeps its state in memory only and uses pickle on the wire, swirld.py:129,160):
 * the engine's whole state -- event columns, can_see table, rounds, witness / fame tables, order -- as one binary file
 * of SoA sections.  sw_load builds a new engine from it (capacity_events 0 = the saved capacity; never less than the
 * saved event count) that continues exactly where the saved one stopped: the same later calls give the same results.
 * sw_save writes version 2 of the format; sw_load also reads version 1, which has no consensus times or rounds received:
 * for the positions such a file had already ordered it reports round received -1 and time NaN (all bits set). */
int sw_save(sw_engine *e, const char *path);
int sw_load(const char *path, int device, int capacity_events, sw_engine **out);

/* ---- several GPUs of one box (one process per GPU), M > 64: ONE hashgraph, identical state and results on every rank,
 * no collective library call on the data path (the reference has no counterpart: it is single-process, swirld.py:331-345):
 *  - can_see: the column tiles of the scan are split over the ranks and every walk stores its row segments straight into
 *    EVERY rank's table over NVLink (P2P stores: the all-gather of the table is fused into the kernel that produces it);
 *  - divide_rounds: the P_r tests of every round step are sharded by member chain; every rank writes its chains' first
 *    hits into every peer's exchange buffer (P2P stores + a system-scope flag) from inside the round kernel.
 * sw_peer_handle writes SW_PEER_HANDLE_BYTES bytes (the CUDA IPC handles of this engine's exchange buffer and can_see
 * table); exchange them out of band (torch.distributed.all_gather_object), then
 * sw_peer_connect(rank, nranks <= 8, handles[nranks][SW_PEER_HANDLE_BYTES]) before the first sw_append.  Every rank must
 * then make the same sw_append / sw_divide_rounds / ... calls. */
#define SW_PEER_HANDLE_BYTES 128
int sw_peer_handle(sw_engine *e, void *handle_out);
int sw_peer_connect(sw_engine *e, int rank, int nranks, const void *handles);

int sw_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SWIRLD_B200_H */
