"""The bytes Engine.new_events signs and hashes for one event (Node.new_event, swirld.py:82-95).

The engine does not parse pickle: the caller pickles with its own Event class, once with a placeholder signature,
and the engine puts the real signature in the placeholder's place.  A pickled bytes object of 64 bytes is its length
and its raw bytes, so the preimage with the real signature is byte for byte dumps(Event(d, p, t, pk, s))."""
from __future__ import annotations

import hashlib
import pickle

SENTINEL = hashlib.sha512(b"swirld_b200 event signature placeholder").digest()


def event_template(event_cls, d, p, t, pk):
    """(msg, pre, sig_at) of the event (d, p, t, pk): msg = dumps((d, p, t, pk)), the signed message; pre =
    dumps(event_cls(d, p, t, pk, SENTINEL)), whose 64 bytes at sig_at are the placeholder."""
    msg = pickle.dumps((d, p, t, pk))
    pre = pickle.dumps(event_cls(d, p, t, pk, SENTINEL))
    at = pre.find(SENTINEL)
    assert at >= 0 and pre.find(SENTINEL, at + 1) < 0, "the placeholder signature must occur exactly once"
    return msg, pre, at
