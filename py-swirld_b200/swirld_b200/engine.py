"""ctypes binding of libswirld_b200.so (include/swirld_b200.h).

There is no CPU implementation behind this module: if the CUDA library is not
built, or no CUDA device is present, construction raises.  The oracle under
oracle/ is test infrastructure and is never imported from here.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libswirld_b200.so")
PEER_HANDLE_BYTES = 128          # SW_PEER_HANDLE_BYTES

SW_E = {-1: "SW_E_ARG", -2: "SW_E_INDEX", -3: "SW_E_KEY", -4: "SW_E_CUDA", -5: "SW_E_CAPACITY",
        -6: "SW_E_PARENT", -7: "SW_E_FORK", -8: "SW_E_UNSUPPORTED"}

# every symbol include/swirld_b200.h declares (tests check the library exports them all)
SYMBOLS = [
    "sw_create", "sw_destroy", "sw_reset", "sw_rewind", "sw_event_record", "sw_event_elapsed_ms", "sw_last_error", "sw_append", "sw_divide_rounds",
    "sw_decide_fame", "sw_find_order", "sw_n_events", "sw_n_divided", "sw_max_round",
    "sw_n_transactions", "sw_get_round", "sw_get_witness_flags", "sw_get_famous", "sw_get_can_see",
    "sw_get_witness_table", "sw_get_consensus", "sw_get_transactions", "sw_get_idx", "sw_get_height",
    "sw_sync", "sw_stats", "sw_flush_l2", "sw_version", "sw_debug_counters", "sw_rc_step_log", "sw_peer_handle", "sw_peer_connect",
    "sw_save", "sw_load", "sw_members", "sw_ingest", "sw_lookup", "sw_batch_divide_rounds",
    "sw_batch_decide_fame", "sw_batch_find_order", "sw_batch_append",
    "sw_get_consensus_times", "sw_get_rounds_received", "sw_find_order_out", "sw_batch_find_order_out",
    "sw_set_member_keys", "sw_verify_events", "sw_ingest_verified", "sw_batch_ingest_verified",
    "sw_get_ids", "sw_sync_summary", "sw_sync_reply", "sw_batch_sync_summary", "sw_batch_sync_reply",
    "sw_set_signing_key", "sw_new_events", "sw_batch_new_events",
]

REPLY_CAP = 4096      # the rows a sync reply is given room for per view, before the one retry at the exact count


class SwStats(C.Structure):
    _fields_ = [("ms_divide_rounds", C.c_double), ("ms_decide_fame", C.c_double),
                ("ms_find_order", C.c_double), ("ms_can_see", C.c_double),
                ("kernel_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("events", C.c_int64), ("events_divided", C.c_int64), ("ms_rounds_kernel", C.c_double),
                ("rounds_cluster_launches", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class EngineError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("%s (%d): %s" % (SW_E.get(code, "SW_E_?"), code, msg))
        self.code = code


_lib = None


def load_library(path: str = LIB_PATH):
    """dlopen the CUDA library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise RuntimeError(
            "%s is missing: build it with `python -m swirld_b200.build` (nvcc, sm_90a). "
            "This engine has no CPU fallback." % path)
    L = C.CDLL(path)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    P = C.POINTER
    L.sw_create.argtypes = [i32, i32, P(C.c_int64), i32, i32, P(vp)]
    L.sw_destroy.argtypes = [vp]; L.sw_destroy.restype = None
    L.sw_reset.argtypes = [vp]
    L.sw_rewind.argtypes = [vp]
    L.sw_event_record.argtypes = [vp, i32]
    L.sw_event_elapsed_ms.argtypes = [vp, i32, i32, P(C.c_double)]
    L.sw_last_error.argtypes = [vp]; L.sw_last_error.restype = C.c_char_p
    L.sw_append.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    L.sw_divide_rounds.argtypes = [vp, i32, i32]
    L.sw_decide_fame.argtypes = [vp, vp, i32]
    L.sw_find_order.argtypes = [vp, vp, i32]
    for f in ("sw_n_events", "sw_n_divided", "sw_max_round", "sw_n_transactions", "sw_sync"):
        getattr(L, f).argtypes = [vp]
    for f in ("sw_get_round", "sw_get_witness_flags", "sw_get_famous", "sw_get_can_see",
              "sw_get_witness_table", "sw_get_transactions", "sw_get_idx", "sw_get_height",
              "sw_get_consensus_times", "sw_get_rounds_received"):
        getattr(L, f).argtypes = [vp, i32, i32, vp]
    L.sw_get_consensus.argtypes = [vp, vp, i32]
    L.sw_stats.argtypes = [vp, P(SwStats)]
    L.sw_flush_l2.argtypes = [vp, i64]
    L.sw_version.argtypes = []
    L.sw_debug_counters.argtypes = [vp, vp, i32]
    L.sw_rc_step_log.argtypes = [vp, vp, i64, i32]
    L.sw_peer_handle.argtypes = [vp, vp]
    L.sw_peer_connect.argtypes = [vp, i32, i32, vp]
    L.sw_members.argtypes = [vp]
    L.sw_ingest.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp]
    L.sw_lookup.argtypes = [vp, i32, vp, vp]
    L.sw_set_member_keys.argtypes = [vp, vp]
    L.sw_verify_events.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.sw_ingest_verified.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.sw_batch_divide_rounds.argtypes = [vp, i32, vp, vp]
    L.sw_batch_decide_fame.argtypes = [vp, i32, vp, i32, vp]
    L.sw_batch_find_order.argtypes = [vp, i32, vp, vp, vp]
    L.sw_find_order_out.argtypes = [vp, vp, i32, vp, vp, vp, i32]
    L.sw_batch_find_order_out.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, i32]
    L.sw_batch_append.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp]
    L.sw_batch_ingest_verified.argtypes = [vp, i32] + [vp] * 14
    L.sw_get_ids.argtypes = [vp, i32, i32, vp]
    L.sw_sync_summary.argtypes = [vp, i32, vp]
    L.sw_sync_reply.argtypes = [vp, i32, vp, i32] + [vp] * 8
    L.sw_batch_sync_summary.argtypes = [vp, i32, vp, vp]
    L.sw_batch_sync_reply.argtypes = [vp, i32, vp, vp, i32] + [vp] * 9
    L.sw_set_signing_key.argtypes = [vp, i32, vp]
    L.sw_new_events.argtypes = [vp, i32] + [vp] * 11
    L.sw_batch_new_events.argtypes = [vp, i32] + [vp] * 13
    L.sw_save.argtypes = [vp, C.c_char_p]
    L.sw_load.argtypes = [C.c_char_p, i32, i32, P(vp)]
    _lib = L
    return L


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _packed(items):
    """A sequence of bytes as (their concatenation, n+1 int64 offsets)."""
    items = [bytes(b) for b in items]
    off = np.zeros(len(items) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in items])
    cat = np.frombuffer(b"".join(items), np.uint8) if off[-1] else np.zeros(1, np.uint8)
    return np.ascontiguousarray(cat), off


class Engine:
    """One node-view of the hashgraph on one GPU; thin, index-space."""

    def __init__(self, M: int, capacity: int, stake=None, coin_period: int = 6, device: int = 0):
        self._lib = load_library()
        self.M, self.capacity = int(M), int(capacity)
        h = C.c_void_p()
        st = None
        if stake is not None:
            arr = (C.c_int64 * M)(*[int(s) for s in stake])
            st = C.cast(arr, C.POINTER(C.c_int64))
        rc = self._lib.sw_create(M, capacity, st, coin_period, device, C.byref(h))
        if rc < 0:
            raise EngineError(rc, (self._lib.sw_last_error(None) or b"").decode())
        self._h = h

    # -- checkpoint / resume
    def save(self, path: str):
        self._chk(self._lib.sw_save(self._h, os.fsencode(path)))

    @classmethod
    def load(cls, path: str, device: int = 0, capacity: int = 0) -> "Engine":
        lib = load_library()
        h = C.c_void_p()
        rc = lib.sw_load(os.fsencode(path), device, capacity, C.byref(h))
        if rc < 0:
            raise EngineError(rc, (lib.sw_last_error(None) or b"").decode())
        self = cls.__new__(cls)
        self._lib, self._h = lib, h
        self.M = self._chk(lib.sw_members(h))
        self.capacity = capacity
        return self

    # -- life cycle
    def close(self):
        if getattr(self, "_h", None):
            self._lib.sw_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _error(self, rc):
        """The exception the single call would raise for the SW_E_* code rc."""
        msg = (self._lib.sw_last_error(self._h) or b"").decode()
        if rc == -2:
            return IndexError(msg)
        if rc == -3:
            return KeyError(msg)
        return EngineError(rc, msg)

    def _chk(self, rc):
        if rc < 0:
            raise self._error(rc)
        return rc

    def reset(self):
        self._chk(self._lib.sw_reset(self._h))

    def rewind(self):
        self._chk(self._lib.sw_rewind(self._h))

    def record(self, slot):
        self._chk(self._lib.sw_event_record(self._h, slot))

    def elapsed_ms(self, a, b):
        ms = C.c_double()
        self._chk(self._lib.sw_event_elapsed_ms(self._h, a, b, C.byref(ms)))
        return ms.value

    # -- the path
    def append(self, p0, p1, creator, t, sig):
        p0 = np.ascontiguousarray(p0, np.int32); p1 = np.ascontiguousarray(p1, np.int32)
        creator = np.ascontiguousarray(creator, np.int32); t = np.ascontiguousarray(t, np.float64)
        sig = np.ascontiguousarray(sig, np.uint8)
        n = p0.shape[0]
        assert p1.shape[0] == n and creator.shape[0] == n and t.shape[0] == n and sig.size == 64 * n
        self._chk(self._lib.sw_append(self._h, n, _ptr(p0), _ptr(p1), _ptr(creator), _ptr(t), _ptr(sig)))

    def ingest(self, ids, p0_ids, p1_ids, creator, t, sig, msgs=None, preimages=None):
        """sw_ingest: events named by 32-byte ids (parents by id, zeros = none), any order; returns the arrival index
        of every input event (-1 = rejected) and the number appended.  With msgs (the signed bytes, dumps(ev[:-1])) and
        preimages (dumps(ev), whose BLAKE2b is the id) it is sw_ingest_verified: a new event whose signature or id
        fails on the GPU is rejected too, with whatever depends on it."""
        ids = np.ascontiguousarray(ids, np.uint8).reshape(-1, 32)
        n = ids.shape[0]
        p0_ids = np.ascontiguousarray(p0_ids, np.uint8).reshape(n, 32)
        p1_ids = np.ascontiguousarray(p1_ids, np.uint8).reshape(n, 32)
        creator = np.ascontiguousarray(creator, np.int32); t = np.ascontiguousarray(t, np.float64)
        sig = np.ascontiguousarray(sig, np.uint8).reshape(n, 64)
        out = np.empty(n, np.int32)
        if msgs is not None and preimages is not None:
            assert len(msgs) == n and len(preimages) == n
            (msg, moff), (pre, poff) = _packed(msgs), _packed(preimages)
            m = self._chk(self._lib.sw_ingest_verified(self._h, n, _ptr(ids), _ptr(p0_ids), _ptr(p1_ids), _ptr(creator),
                                                       _ptr(t), _ptr(sig), _ptr(msg), _ptr(moff), _ptr(pre), _ptr(poff),
                                                       _ptr(out)))
            return out, m
        m = self._chk(self._lib.sw_ingest(self._h, n, _ptr(ids), _ptr(p0_ids), _ptr(p1_ids), _ptr(creator), _ptr(t), _ptr(sig), _ptr(out)))
        return out, m

    def set_member_keys(self, pks):
        """sw_set_member_keys: the members' Ed25519 public keys, an (M, 32) uint8 array or M values of 32 bytes."""
        if isinstance(pks, np.ndarray):
            a = np.ascontiguousarray(pks, np.uint8).reshape(-1)
        else:
            a = np.frombuffer(b"".join(bytes(p) for p in pks), np.uint8).copy()
        assert a.size == 32 * self.M, "need %d keys of 32 bytes" % self.M
        self._chk(self._lib.sw_set_member_keys(self._h, _ptr(a)))

    def verify_events(self, creator, sig, msgs, preimages, ids):
        """sw_verify_events: per event, bit 0 = sig is creator's valid Ed25519 signature of msgs[i] (libsodium's
        verdict), bit 1 = BLAKE2b-256(preimages[i]) == ids[i].  Returns the flags as a uint8 array."""
        creator = np.ascontiguousarray(creator, np.int32)
        n = creator.shape[0]
        sig = np.ascontiguousarray(sig, np.uint8).reshape(n, 64) if n else np.zeros((1, 64), np.uint8)
        ids = np.ascontiguousarray(ids, np.uint8).reshape(n, 32) if n else np.zeros((1, 32), np.uint8)
        assert len(msgs) == n and len(preimages) == n
        (msg, moff), (pre, poff) = _packed(msgs), _packed(preimages)
        out = np.zeros(max(n, 1), np.uint8)
        self._chk(self._lib.sw_verify_events(self._h, n, _ptr(creator), _ptr(sig), _ptr(msg), _ptr(moff), _ptr(pre),
                                             _ptr(poff), _ptr(ids), _ptr(out)))
        return out[:n]

    def set_signing_key(self, member, sk):
        """sw_set_signing_key: this view signs its new events as `member` with libsodium's 64-byte secret key (seed ||
        pk); pk must be member's key in set_member_keys.  Only the expanded key is kept, in device memory."""
        sk = bytes(sk)
        assert len(sk) == 64, "libsodium's secret key is 64 bytes"
        buf = C.create_string_buffer(sk, 64)
        try:
            self._chk(self._lib.sw_set_signing_key(self._h, int(member), C.cast(buf, C.c_void_p)))
        finally:
            C.memset(buf, 0, 64)

    def new_events(self, templates, p0_ids=None, p1_ids=None, t=None, ingest=True):
        """sw_new_events: sign and hash events of this view's signing member.  templates[i] = (msg, pre, sig_at) as
        events.event_template makes them.  Returns (sig, ids) as (n, 64) and (n, 32) uint8 arrays; with ingest (p0_ids,
        p1_ids and t given) also enters the events as Engine.ingest would: (sig, ids, index_out, appended)."""
        n = len(templates)
        msg, moff, pre, poff, at = _templates(templates)
        sig, ids = np.zeros((max(n, 1), 64), np.uint8), np.zeros((max(n, 1), 32), np.uint8)
        if not ingest:
            self._chk(self._lib.sw_new_events(self._h, n, None, None, None, _ptr(msg), _ptr(moff), _ptr(pre), _ptr(poff),
                                              _ptr(at), _ptr(sig), _ptr(ids), None))
            return sig[:n], ids[:n]
        p0 = np.ascontiguousarray(p0_ids, np.uint8).reshape(n, 32)
        p1 = np.ascontiguousarray(p1_ids, np.uint8).reshape(n, 32)
        t = np.ascontiguousarray(t, np.float64).reshape(n)
        out = np.empty(max(n, 1), np.int32)
        m = self._chk(self._lib.sw_new_events(self._h, n, _ptr(p0), _ptr(p1), _ptr(t), _ptr(msg), _ptr(moff), _ptr(pre),
                                              _ptr(poff), _ptr(at), _ptr(sig), _ptr(ids), _ptr(out)))
        return sig[:n], ids[:n], out[:n], m

    def lookup(self, ids):
        ids = np.ascontiguousarray(ids, np.uint8).reshape(-1, 32)
        out = np.empty(ids.shape[0], np.int32)
        self._chk(self._lib.sw_lookup(self._h, ids.shape[0], _ptr(ids), _ptr(out)))
        return out

    def ids(self, first=0, n=None):
        """sw_get_ids: the 32-byte id of events [first, first+n) as an (n, 32) uint8 array, zeros for an event that has
        none (it came through append, not ingest)."""
        n = self.n_events - first if n is None else n
        out = np.zeros((n, 32), np.uint8)
        if n:
            self._chk(self._lib.sw_get_ids(self._h, first, n, _ptr(out)))
        return out

    def sync_summary(self, head):
        """sw_sync_summary: what this view sends when it asks a peer to sync (swirld.py:125-126), as M heights: of the
        latest event of each member that `head` sees, -1 where it sees none."""
        out = np.empty(self.M, np.int32)
        self._chk(self._lib.sw_sync_summary(self._h, int(head), _ptr(out)))
        return out

    def sync_reply(self, head, summary, rows=True):
        """sw_sync_reply: the events ask_sync (swirld.py:154-161) sends from `head` to a requester whose summary this is,
        in ascending index.  Returns their indices, and with rows (index, (ids, p0_ids, p1_ids, creator, t, sig)):
        the columns Engine.ingest takes.  rows needs every event of the reply to have come through ingest."""
        summary = np.ascontiguousarray(summary, np.int32)
        assert summary.shape == (self.M,)
        cap = min(int(head) + 1, REPLY_CAP)
        for attempt in range(2):
            idx = np.empty(max(cap, 1), np.int32)
            cols = _reply_columns(cap) if rows else None
            cnt = C.c_int32(0)
            rc = self._lib.sw_sync_reply(self._h, int(head), _ptr(summary), cap, _ptr(idx), C.byref(cnt),
                                         *[_ptr(a) if rows else None for a in (cols or [None] * 6)])
            if rc == -5 and attempt == 0:                  # SW_E_CAPACITY: cnt holds the exact count
                cap = cnt.value
                continue
            n = self._chk(rc)
            break
        if not rows:
            return idx[:n]
        return idx[:n], tuple(a[:n] for a in cols)

    def append_trace(self, tr, first=0, n=None):
        n = tr.N - first if n is None else n
        s = slice(first, first + n)
        self.append(tr.p0[s], tr.p1[s], tr.creator[s], tr.t[s], tr.sig[s])

    def divide_rounds(self, first, n):
        self._chk(self._lib.sw_divide_rounds(self._h, first, n))

    def decide_fame(self):
        cap = max(64, self.n_divided + 2)
        if getattr(self, "_newc_buf", None) is None or self._newc_buf.size < cap:
            self._newc_buf = np.empty(cap, np.int32)
        n = self._chk(self._lib.sw_decide_fame(self._h, _ptr(self._newc_buf), self._newc_buf.size))
        return self._newc_buf[:n].tolist()

    def find_order(self, new_c):
        a = np.ascontiguousarray(sorted(new_c), np.int32)
        if a.size == 0:
            return 0
        return self._chk(self._lib.sw_find_order(self._h, _ptr(a), a.size))

    def find_order_out(self, new_c):
        """find_order, returning what it appended to the order: (events, consensus times, rounds received), the
        parallel arrays transactions() / consensus_times() / rounds_received() gain, from the copy find_order makes
        anyway."""
        a = np.ascontiguousarray(sorted(new_c), np.int32)
        cap = max(0, self.n_divided - self.n_transactions)
        ev, ts, rr = np.empty(cap, np.int32), np.empty(cap, np.float64), np.empty(cap, np.int32)
        n = self._chk(self._lib.sw_find_order_out(self._h, _ptr(a), a.size, _ptr(ev), _ptr(ts), _ptr(rr), cap))
        return ev[:n].copy(), ts[:n].copy(), rr[:n].copy()

    # -- views
    @property
    def n_events(self):
        return self._lib.sw_n_events(self._h)

    @property
    def n_divided(self):
        return self._lib.sw_n_divided(self._h)

    @property
    def n_transactions(self):
        return self._lib.sw_n_transactions(self._h)

    @property
    def max_round(self):
        return self._chk(self._lib.sw_max_round(self._h))

    def _get(self, fn, dtype, first, n, width=1):
        out = np.empty((n, width) if width > 1 else n, dtype)
        if n:
            self._chk(fn(self._h, first, n, _ptr(out)))
        return out

    def rounds(self, first=0, n=None):
        return self._get(self._lib.sw_get_round, np.int32, first, self.n_divided - first if n is None else n)

    def witness_flags(self, first=0, n=None):
        return self._get(self._lib.sw_get_witness_flags, np.uint8, first, self.n_divided - first if n is None else n)

    def famous(self, first=0, n=None):
        return self._get(self._lib.sw_get_famous, np.int8, first, self.n_events - first if n is None else n)

    def can_see(self, first=0, n=None):
        n = self.n_divided - first if n is None else n
        out = np.empty((n, self.M), np.int32)
        if n:
            self._chk(self._lib.sw_get_can_see(self._h, first, n, _ptr(out)))
        return out

    def witness_table(self, first_round=0, n_rounds=None):
        n_rounds = self.max_round + 1 - first_round if n_rounds is None else n_rounds
        out = np.empty((n_rounds, self.M), np.int32)
        if n_rounds:
            self._chk(self._lib.sw_get_witness_table(self._h, first_round, n_rounds, _ptr(out)))
        return out

    def consensus(self):
        buf = np.empty(max(1, self.max_round + 2), np.int32)
        n = self._chk(self._lib.sw_get_consensus(self._h, _ptr(buf), buf.size))
        return buf[:n].copy()

    def transactions(self, first=0, n=None):
        return self._get(self._lib.sw_get_transactions, np.int32, first, self.n_transactions - first if n is None else n)

    def consensus_times(self, first=0, n=None):
        """The consensus timestamp (swirld.py:305) of transactions()[first:first+n]."""
        return self._get(self._lib.sw_get_consensus_times, np.float64, first, self.n_transactions - first if n is None else n)

    def rounds_received(self, first=0, n=None):
        """The round received (the round whose find_order step ordered it, swirld.py:283) of transactions()[first:first+n]."""
        return self._get(self._lib.sw_get_rounds_received, np.int32, first, self.n_transactions - first if n is None else n)

    def idx(self, first=0, n=None):
        return self._get(self._lib.sw_get_idx, np.int32, first, self.n_events - first if n is None else n)

    def heights(self, first=0, n=None):
        return self._get(self._lib.sw_get_height, np.int32, first, self.n_events - first if n is None else n)

    def sync(self):
        self._chk(self._lib.sw_sync(self._h))

    def stats(self):
        s = SwStats()
        self._chk(self._lib.sw_stats(self._h, C.byref(s)))
        return s.as_dict()

    def debug_counters(self, clear=True):
        out = np.zeros(16, np.int64)
        self._chk(self._lib.sw_debug_counters(self._h, _ptr(out), 1 if clear else 0))
        return out

    def rc_step_log(self, clear=True):
        """The cluster round kernel's step log (engine created with SW_RC_STEPS set): [steps, 16 CTAs, 16] uint32 in
        cycles, fields in swirld_rcluster.cuh's RL_* order."""
        n = self._chk(self._lib.sw_rc_step_log(self._h, None, 0, 0))
        out = np.zeros(16 + n * 16 * 16, np.uint32)
        self._chk(self._lib.sw_rc_step_log(self._h, _ptr(out), out.size, 1 if clear else 0))
        kept = min(n, int(out[1]))
        return out[16:16 + kept * 256].reshape(kept, 16, 16)

    # -- several GPUs of one box, M > 64 (include/swirld_b200.h: sw_peer_handle / sw_peer_connect)
    def peer_handle(self) -> bytes:
        """The CUDA IPC handles (PEER_HANDLE_BYTES bytes) of this engine's exchange buffer and can_see table."""
        buf = C.create_string_buffer(PEER_HANDLE_BYTES)
        self._chk(self._lib.sw_peer_handle(self._h, C.cast(buf, C.c_void_p)))
        return buf.raw

    def peer_connect(self, rank: int, nranks: int, handles: bytes):
        """handles = the nranks handles concatenated in rank order; call before the first divide_rounds."""
        assert len(handles) == PEER_HANDLE_BYTES * nranks
        buf = C.create_string_buffer(handles, len(handles))
        self._chk(self._lib.sw_peer_connect(self._h, rank, nranks, C.cast(buf, C.c_void_p)))

    def flush_l2(self, nbytes=256 << 20):
        self._chk(self._lib.sw_flush_l2(self._h, nbytes))

    def results(self):
        """Same dict as oracle.Oracle.results() (index space)."""
        return {"round": self.rounds(), "witness": self.witness_flags(),
                "witness_table": self.witness_table(), "famous": self.famous(),
                "consensus": self.consensus(), "transactions": self.transactions()}


def batch_divide_rounds(engines, firsts, counts):
    """sw_batch_divide_rounds: divide_rounds of several independent node-views (one member count, one kernel family,
    one device) in one call.  Calls of at most 16 events run in one launch for all views at any M, whatever their
    stakes; larger calls need M <= 64 and one stake shape among them, else the whole call is refused."""
    B = len(engines)
    arr = (C.c_void_p * B)(*[e._h for e in engines])
    f = np.ascontiguousarray(firsts, np.int32)
    n = np.ascontiguousarray(counts, np.int32)
    engines[0]._chk(engines[0]._lib.sw_batch_divide_rounds(C.cast(arr, C.c_void_p), B, _ptr(f), _ptr(n)))


def _handles(engines):
    arr = (C.c_void_p * len(engines))(*[e._h for e in engines])
    return C.cast(arr, C.c_void_p)


def _per_view(what, engines, results, counts):
    """Raise the views' own failures, after the whole batch has run, as one ExceptionGroup: each member is what the
    single call would have raised, with .view set; the group's .results holds every view's result (None: failed)."""
    errs = []
    for v, rc in enumerate(counts):
        if rc < 0:
            ex = engines[v]._error(int(rc))
            ex.view = v
            errs.append(ex)
            results[v] = None
    if errs:
        g = ExceptionGroup("%s: %d of %d views failed" % (what, len(errs), len(engines)), errs)
        g.results = results
        raise g
    return results


def batch_decide_fame(engines):
    """sw_batch_decide_fame: decide_fame of several node-views (one member count, one kernel family, one device) in one
    call.  Returns each view's new consensus rounds, as Engine.decide_fame does.  Argument errors raise at once;
    failures the device finds in some views raise as an ExceptionGroup after every view has run (see _per_view)."""
    B = len(engines)
    if B == 0:
        return []
    cap = max(max(64, e.n_divided + 2) for e in engines)      # as Engine.decide_fame chooses it, for the largest view
    out = np.empty((B, cap), np.int32)
    cnt = np.zeros(B, np.int32)
    rc = engines[0]._lib.sw_batch_decide_fame(_handles(engines), B, _ptr(out), cap, _ptr(cnt))
    if rc < 0 and not (cnt < 0).any():
        engines[0]._chk(rc)                # refused as a whole: nothing ran, count_out was not written
    return _per_view("batch_decide_fame", engines, [out[v, :max(0, int(n))].tolist() for v, n in enumerate(cnt)], cnt)


def batch_append(engines, columns):
    """sw_batch_append: Engine.append of several node-views (one device) in one call; columns[v] = (p0, p1, creator,
    t, sig) of view v.  Returns the events each view appended.  Argument errors raise at once; a view whose events
    append would refuse appends nothing, and those failures raise as an ExceptionGroup after every view has appended
    (see _per_view)."""
    B = len(engines)
    assert len(columns) == B
    if B == 0:
        return []
    cols = [[np.asarray(c) for c in view] for view in columns]
    ns = [len(c[0]) for c in cols]
    for c, n in zip(cols, ns):
        assert len(c[1]) == n and len(c[2]) == n and len(c[3]) == n and c[4].size == 64 * n
    cat = [np.ascontiguousarray(np.concatenate([c[k].reshape(-1) for c in cols]), dt)
           for k, dt in enumerate((np.int32, np.int32, np.int32, np.float64, np.uint8))]
    offs = np.zeros(B + 1, np.int32)
    offs[1:] = np.cumsum(ns)
    rcs = np.zeros(B, np.int32)
    rc = engines[0]._lib.sw_batch_append(_handles(engines), B, _ptr(offs), *[_ptr(a) for a in cat], _ptr(rcs))
    if rc < 0 and not (rcs < 0).any():
        engines[0]._chk(rc)                # refused as a whole: nothing ran, rc_out was not written
    return _per_view("batch_append", engines, list(ns), rcs)


def batch_ingest(engines, batches):
    """sw_batch_ingest_verified: Engine.ingest with msgs and preimages for several node-views (one device) in one call;
    batches[v] = (ids, p0_ids, p1_ids, creator, t, sig, msgs, preimages) of view v.  Every event the views would verify
    is verified once on the GPU, however many views receive it.  Returns ([(index_out, appended) per view], the number
    of events verified).  Argument errors raise at once; a view whose batch is not a DAG or that runs out of capacity
    ingests nothing, and those failures raise as an ExceptionGroup after every other view has ingested (see
    _per_view; the group's .n_verified holds the count)."""
    B = len(engines)
    assert len(batches) == B
    if B == 0:
        return [], 0
    cols, msgs, pres = [], [], []
    for ids, p0_ids, p1_ids, creator, t, sig, m, p in batches:
        ids = np.asarray(ids, np.uint8).reshape(-1, 32)
        n = ids.shape[0]
        cols.append((ids, np.asarray(p0_ids, np.uint8).reshape(n, 32), np.asarray(p1_ids, np.uint8).reshape(n, 32),
                     np.asarray(creator, np.int32).reshape(n), np.asarray(t, np.float64).reshape(n),
                     np.asarray(sig, np.uint8).reshape(n, 64)))
        assert len(m) == n and len(p) == n
        msgs += list(m)
        pres += list(p)
    ns = [c[0].shape[0] for c in cols]
    cat = [np.ascontiguousarray(np.concatenate([c[k] for c in cols]).reshape(-1)) for k in range(6)]
    (msg, moff), (pre, poff) = _packed(msgs), _packed(pres)
    offs = np.zeros(B + 1, np.int32)
    offs[1:] = np.cumsum(ns)
    out = np.empty(max(1, int(offs[-1])), np.int32)
    cnt = np.zeros(B, np.int32)
    nv = C.c_int32(0)
    rc = engines[0]._lib.sw_batch_ingest_verified(_handles(engines), B, _ptr(offs), *[_ptr(a) for a in cat], _ptr(msg),
                                                  _ptr(moff), _ptr(pre), _ptr(poff), _ptr(out), _ptr(cnt), C.byref(nv))
    if rc < 0 and not (cnt < 0).any():
        engines[0]._chk(rc)                # refused as a whole: nothing ran, count_out was not written
    res = [(out[a:b].copy(), int(m)) for a, b, m in zip(offs[:-1].tolist(), offs[1:].tolist(), cnt)]
    try:
        return _per_view("batch_ingest", engines, res, cnt), nv.value
    except ExceptionGroup as g:
        g.n_verified = nv.value
        raise


def _templates(templates):
    """(msg, msg_off, pre, pre_off, sig_at) of (msg, pre, sig_at) triples, as sw_new_events takes them."""
    (msg, moff), (pre, poff) = _packed([m for m, _, _ in templates]), _packed([p for _, p, _ in templates])
    at = np.ascontiguousarray([a for _, _, a in templates] or [0], np.int64)
    return msg, moff, pre, poff, at


def batch_new_events(engines, templates, p0_ids=None, p1_ids=None, t=None, ingest=True):
    """sw_batch_new_events: Engine.new_events of several node-views (one device) in one call, every event signed in one
    launch.  templates[v] lists view v's (msg, pre, sig_at); with ingest, p0_ids[v], p1_ids[v] and t[v] are its columns.
    Returns [(sig, ids)] per view, or with ingest [(sig, ids, index_out, appended)].  Argument errors raise at once; a
    view's own failure raises as an ExceptionGroup after every other view has ingested (see _per_view)."""
    B = len(engines)
    assert len(templates) == B
    if B == 0:
        return []
    ns = [len(x) for x in templates]
    offs = np.zeros(B + 1, np.int32)
    offs[1:] = np.cumsum(ns)
    N = int(offs[-1])
    msg, moff, pre, poff, at = _templates([x for view in templates for x in view])
    sig, ids = np.zeros((max(N, 1), 64), np.uint8), np.zeros((max(N, 1), 32), np.uint8)
    ab = list(zip(offs[:-1].tolist(), offs[1:].tolist()))
    L = engines[0]._lib
    if not ingest:
        engines[0]._chk(L.sw_batch_new_events(_handles(engines), B, _ptr(offs), None, None, None, _ptr(msg), _ptr(moff),
                                              _ptr(pre), _ptr(poff), _ptr(at), _ptr(sig), _ptr(ids), None, None))
        return [(sig[a:b], ids[a:b]) for a, b in ab]
    cat = lambda cols, shape, dt: np.ascontiguousarray(
        np.concatenate([np.asarray(c, dt).reshape((n,) + shape) for c, n in zip(cols, ns)]) if N else np.zeros((1,) + shape, dt))
    p0, p1, tt = cat(p0_ids, (32,), np.uint8), cat(p1_ids, (32,), np.uint8), cat(t, (), np.float64)
    out = np.empty(max(N, 1), np.int32)
    cnt = np.zeros(B, np.int32)
    rc = L.sw_batch_new_events(_handles(engines), B, _ptr(offs), _ptr(p0), _ptr(p1), _ptr(tt), _ptr(msg), _ptr(moff),
                               _ptr(pre), _ptr(poff), _ptr(at), _ptr(sig), _ptr(ids), _ptr(out), _ptr(cnt))
    if rc < 0 and not (cnt < 0).any():
        engines[0]._chk(rc)                # refused as a whole: nothing ran, count_out was not written
    res = [(sig[a:b], ids[a:b], out[a:b].copy(), int(m)) for (a, b), m in zip(ab, cnt)]
    return _per_view("batch_new_events", engines, res, cnt)


def _reply_columns(n):
    """Room for n rows in sw_ingest's layout: ids, p0_ids, p1_ids, creator, t, sig."""
    n = max(n, 1)
    return [np.empty((n, 32), np.uint8), np.empty((n, 32), np.uint8), np.empty((n, 32), np.uint8),
            np.empty(n, np.int32), np.empty(n, np.float64), np.empty((n, 64), np.uint8)]


def batch_sync_summary(engines, heads):
    """sw_batch_sync_summary: Engine.sync_summary of several node-views (one device, any member counts) in one call.
    Returns each view's summary."""
    B = len(engines)
    assert len(heads) == B
    if B == 0:
        return []
    h = np.ascontiguousarray(heads, np.int32)
    offs = np.cumsum([0] + [e.M for e in engines])
    out = np.empty(max(1, int(offs[-1])), np.int32)
    engines[0]._chk(engines[0]._lib.sw_batch_sync_summary(_handles(engines), B, _ptr(h), _ptr(out)))
    return [out[a:b] for a, b in zip(offs[:-1], offs[1:])]


def batch_sync_reply(engines, heads, summaries, rows=True):
    """sw_batch_sync_reply: Engine.sync_reply of several node-views (one device, any member counts) in one call.
    Returns each view's indices, and with rows (indices, columns): columns[v] = view v's (ids, p0_ids, p1_ids,
    creator, t, sig), slices of one concatenation laid out as batch_ingest (sw_batch_ingest_verified) takes it."""
    B = len(engines)
    assert len(heads) == B and len(summaries) == B
    if B == 0:
        return ([], []) if rows else []
    h = np.ascontiguousarray(heads, np.int32)
    for e, s in zip(engines, summaries):
        assert len(s) == e.M
    S = np.ascontiguousarray(np.concatenate([np.asarray(s, np.int32) for s in summaries]), np.int32)
    cap = int(min(sum(int(x) + 1 for x in heads), REPLY_CAP * B))
    offs, cnt = np.zeros(B + 1, np.int32), np.zeros(B, np.int32)
    for attempt in range(2):
        idx = np.empty(max(cap, 1), np.int32)
        cols = _reply_columns(cap) if rows else None
        rc = engines[0]._lib.sw_batch_sync_reply(_handles(engines), B, _ptr(h), _ptr(S), cap, _ptr(offs), _ptr(cnt),
                                                 _ptr(idx), *[_ptr(a) if rows else None for a in (cols or [None] * 6)])
        if rc == -5 and attempt == 0:                      # SW_E_CAPACITY: cnt holds the exact counts
            cap = int(cnt.sum())
            continue
        engines[0]._chk(rc)
        break
    ab = list(zip(offs[:-1].tolist(), offs[1:].tolist()))
    index = [idx[a:b] for a, b in ab]
    if not rows:
        return index
    return index, [tuple(c[a:b] for c in cols) for a, b in ab]


def batch_find_order(engines, new_cs):
    """sw_batch_find_order: find_order(new_cs[v]) of every view in one call.  Returns the events each view appended
    to its order; errors as batch_decide_fame."""
    B = len(engines)
    assert len(new_cs) == B
    if B == 0:
        return []
    flat = np.ascontiguousarray(np.concatenate([np.asarray(sorted(nc), np.int32) for nc in new_cs]), np.int32)
    offs = np.zeros(B + 1, np.int32)
    offs[1:] = np.cumsum([len(nc) for nc in new_cs])
    cnt = np.zeros(B, np.int32)
    rc = engines[0]._lib.sw_batch_find_order(_handles(engines), B, _ptr(flat), _ptr(offs), _ptr(cnt))
    if rc < 0 and not (cnt < 0).any():
        engines[0]._chk(rc)
    return _per_view("batch_find_order", engines, [int(n) for n in cnt], cnt)


def batch_find_order_out(engines, new_cs):
    """sw_batch_find_order_out: batch_find_order, returning each view's (events, consensus times, rounds received), as
    Engine.find_order_out does, from the one copy the batched call makes; errors as batch_find_order."""
    B = len(engines)
    assert len(new_cs) == B
    if B == 0:
        return []
    flat = np.ascontiguousarray(np.concatenate([np.asarray(sorted(nc), np.int32) for nc in new_cs]), np.int32)
    offs = np.zeros(B + 1, np.int32)
    offs[1:] = np.cumsum([len(nc) for nc in new_cs])
    cnt = np.zeros(B, np.int32)
    cap = sum(max(0, e.n_divided - e.n_transactions) for e in engines)
    ev, ts, rr = np.empty(cap, np.int32), np.empty(cap, np.float64), np.empty(cap, np.int32)
    oo = np.zeros(B + 1, np.int32)
    rc = engines[0]._lib.sw_batch_find_order_out(_handles(engines), B, _ptr(flat), _ptr(offs), _ptr(cnt),
                                                 _ptr(ev), _ptr(ts), _ptr(rr), _ptr(oo), cap)
    if rc < 0 and not (cnt < 0).any():
        engines[0]._chk(rc)
    none = (ev[:0], ts[:0], rr[:0])
    out = [(ev[a:b], ts[a:b], rr[a:b]) if b > a else none for a, b in zip(oo[:-1].tolist(), oo[1:].tolist())]
    return _per_view("batch_find_order_out", engines, out, cnt)


def run_engine(tr, K, stake=None, coin_period=6, device=0, find_order=True):
    """Feed a trace with the call schedule K; returns results() + new_c per call."""
    from .traces import chunks
    e = Engine(tr.M, tr.N, stake, coin_period, device)
    ncs = []
    for first, cnt in chunks(tr.N, K):
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        if find_order:
            e.find_order(nc)
        ncs.append(sorted(nc))
    res = e.results()
    res["new_c_per_call"] = ncs
    res["can_see"] = e.can_see()
    res["stats"] = e.stats()
    res["engine"] = e
    return res
