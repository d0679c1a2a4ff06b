"""Prefetch for compressed-resident modules: decode the next module's weights on a side stream while the current
module computes.

`compress_module(model, prefetch=True)` gives the root module one `Prefetcher`.  Its decisions (which output slot a
module reads, which stream waits for which, what is pending) are plain Python here; the CUDA calls sit behind a small
ops interface (`CudaOps`), so that the host tests drive the same class with fake streams and events.

Two output slots: slot 0 is the buffer the plans were created with, slot 1 one more of its size.  Every decode runs
on the side stream (`DecodePlan.run_into`, a CTA-budgeted single launch), so all runs that share the plans' scratch
stay ordered on one stream.  Within one forward of the root module, module m's successor is learned (the module whose
pre-hook came next the last time), and at m's pre-hook that successor is decoded into the slot m does not read.  A
wrong or missing prediction costs one serial decode; a prediction never crosses root forwards, and the root's forward
hook joins the side stream, so no side-stream work outlives a root forward (a captured root forward joins every fork).
"""
from __future__ import annotations

import os

import torch

# CTAs of a prefetch decode (0: the whole device) and the side stream's priority, from the sweep of
# tools/prefetch_bench.py (DESIGN §3.9): on an H100 every smaller budget was slower, and high priority bought nothing.
DEFAULT_CTAS = 0
PRIORITY = 0


def prefetch_ctas() -> int:
    """The CTA budget of a prefetch decode: ZIPNN_B200_PREFETCH_CTAS, else DEFAULT_CTAS (<= 0: the whole device)."""
    e = os.environ.get("ZIPNN_B200_PREFETCH_CTAS")
    return int(e) if e else DEFAULT_CTAS


class Prefetcher:
    """The scheduling state of one root module.  `ops` provides:
      record_current() -> an event recorded now on the current stream;
      side_wait(event)  -- the side stream waits for it;
      current_wait(event) -- the current stream waits for it;
      decode(key, slot) -> an event recorded on the side stream after decoding module `key` into `slot`
                           (enqueued on the side stream)."""

    def __init__(self, ops):
        self.ops = ops
        self.succ = {}        # module key -> the key whose pre-hook followed it in the last root forward
        self.active = False   # inside a forward of the root module
        self.prev = None      # previous module of this root forward
        self.pending = None   # (key, slot, event) of the prefetch in flight
        self.last = None      # event of the side stream's last decode

    def root_begin(self) -> None:
        self.active, self.prev, self.pending, self.last = True, None, None, None

    def root_end(self) -> None:
        """Join the side stream; nothing is predicted across root forwards."""
        if self.last is not None:
            self.ops.current_wait(self.last)
        self.active, self.prev, self.pending, self.last = False, None, None, None

    def _decode(self, key, slot):
        self.ops.side_wait(self.ops.record_current())   # every earlier reader of `slot` is on the current stream
        ev = self.ops.decode(key, slot)
        self.last = ev
        return ev

    def before(self, key) -> int:
        """Module `key`'s pre-hook: -> the slot whose views it binds, decoded before it runs on the current stream."""
        p, self.pending = self.pending, None
        if p is not None and p[0] == key:
            slot = p[1]
            self.ops.current_wait(p[2])
        else:
            # a wrong prefetch sits earlier on the side stream and every reader earlier on the current one: both
            # slots are free
            slot = 0
            self.ops.current_wait(self._decode(key, slot))
        if self.active:
            if self.prev is not None:
                self.succ[self.prev] = key
            self.prev = key
            n = self.succ.get(key)
            if n is not None:
                self.pending = (n, 1 - slot, self._decode(n, 1 - slot))
        return slot


_SIDE = {}


def side_stream(dev) -> torch.cuda.Stream:
    """The one prefetch stream of device `dev`."""
    s = _SIDE.get(dev)
    if s is None:
        s = _SIDE[dev] = torch.cuda.Stream(device=dev, priority=PRIORITY)
    return s


class CudaOps:
    """The CUDA side of a Prefetcher: `plans[key]` decodes into `slots[slot]` on `side`, `max_ctas` CTAs at most."""

    def __init__(self, dev, plans, slots, max_ctas):
        self.dev, self.plans, self.slots, self.max_ctas = dev, plans, slots, max_ctas
        self.side = side_stream(dev)

    def record_current(self):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        return ev

    def side_wait(self, ev) -> None:
        self.side.wait_event(ev)

    def current_wait(self, ev) -> None:
        torch.cuda.current_stream(self.dev).wait_event(ev)

    def decode(self, key, slot):
        with torch.cuda.stream(self.side):
            self.plans[key].run_into(self.slots[slot], self.max_ctas)
        ev = torch.cuda.Event()
        ev.record(self.side)
        return ev
