"""The prefetch scheduler of compressed-resident modules (zipnn_b200/prefetch.py) without a GPU.

The scheduler is driven the way the module hooks drive it, with fake streams and events that record every operation.
A happens-before graph over those operations (program order on each stream, plus an edge from each recorded event to
every later wait on it) then checks, over fixed and random module sequences:
  * every read of a slot by module m happens after m's decode into that slot, with no later decode of another
    module into that slot ordered before the read;
  * no decode into a slot is concurrent with a read of it;
  * every decode runs on the side stream;
  * the side stream is joined when each root forward ends, and after each call outside a root forward.
Also: the new plan entry point is declared in the header and bound.
"""
import os
import random
import re

import pytest

from zipnn_b200 import _native
from zipnn_b200.prefetch import Prefetcher

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Ops:
    """Two fake streams; every operation is a node, edges are happens-before."""

    def __init__(self):
        self.nodes = []         # (stream, kind, key, slot)
        self.preds = []         # node -> set of direct predecessors
        self.tail = {"cur": None, "side": None}
        self.pending_waits = {"cur": [], "side": []}

    def _add(self, stream, kind, key=None, slot=None):
        i = len(self.nodes)
        self.nodes.append((stream, kind, key, slot))
        p = set(self.pending_waits[stream])
        if self.tail[stream] is not None:
            p.add(self.tail[stream])
        self.preds.append(p)
        self.pending_waits[stream] = []
        self.tail[stream] = i
        return i

    # the ops interface of Prefetcher
    def record_current(self):
        return ("ev", self._add("cur", "record"))

    def side_wait(self, ev):
        self.pending_waits["side"].append(ev[1])

    def current_wait(self, ev):
        self.pending_waits["cur"].append(ev[1])

    def decode(self, key, slot):
        n = self._add("side", "decode", key, slot)
        return ("ev", n)

    # what the test does on the current stream
    def read(self, key, slot):
        return self._add("cur", "read", key, slot)

    def marker(self):
        return self._add("cur", "marker")

    def hb(self, a, b):
        """a happens before b."""
        if a == b:
            return False
        seen, todo = set(), [b]
        while todo:
            x = todo.pop()
            for p in self.preds[x]:
                if p == a:
                    return True
                if p not in seen:
                    seen.add(p)
                    todo.append(p)
        return False

    def check(self, joins):
        decodes = [i for i, n in enumerate(self.nodes) if n[1] == "decode"]
        assert all(self.nodes[i][0] == "side" for i in decodes)
        for r, (st, kind, key, slot) in enumerate(self.nodes):
            if kind != "read":
                continue
            before = [d for d in decodes if self.nodes[d][3] == slot and self.hb(d, r)]
            for d in decodes:
                if self.nodes[d][3] == slot:
                    assert d in before or self.hb(r, d), f"decode {d} into slot {slot} concurrent with read {r}"
            assert before, f"read {r} of slot {slot} by {key} follows no decode"
            last = max(before)   # decodes are all on the side stream: program order is their order
            assert self.nodes[last][2] == key, f"read {r} by {key} sees module {self.nodes[last][2]}'s weights"
        for m in joins:
            assert all(self.hb(d, m) for d in decodes if d < m), f"side stream not joined at {m}"


def drive(script):
    """script: list of ("root", [keys], raise_at or None) and ("direct", key)."""
    ops = Ops()
    s = Prefetcher(ops)
    ops.hits = 0   # pre-hooks that found their module prefetched
    joins = []
    for step in script:
        if step[0] == "root":
            _, keys, raise_at = step
            s.root_begin()
            for j, k in enumerate(keys):
                if raise_at is not None and j == raise_at:
                    break                # the forward raised: the always-called root hook still runs
                ops.hits += s.pending is not None and s.pending[0] == k
                ops.read(k, s.before(k))
            s.root_end()
            joins.append(ops.marker())
        else:
            k = step[1]
            ops.read(k, s.before(k))
            joins.append(ops.marker())
    ops.check(joins)
    return ops, s


def test_steady_repetition_uses_predictions():
    ops, _ = drive([("root", list(range(6)), None)] * 4)
    decodes = [n for n in ops.nodes if n[1] == "decode"]
    # first forward: 6 serial decodes; later ones: 1 serial (the first module) + 5 prefetches, every one used
    assert len(decodes) == 6 + 3 * 6
    assert ops.hits == 3 * 5


def test_changed_order_between_forwards():
    drive([("root", [0, 1, 2, 3], None), ("root", [0, 2, 1, 3], None), ("root", [3, 2, 1, 0], None), ("root", [0, 1, 2, 3], None)])


def test_module_called_twice_in_a_row():
    drive([("root", [0, 1, 1, 2], None)] * 3 + [("root", [0, 1, 2], None), ("root", [0, 1, 1, 1, 2], None)])


def test_skipped_modules():
    drive([("root", [0, 1, 2, 3], None), ("root", [0, 2, 3], None), ("root", [0, 1, 3], None), ("root", [0, 1, 2, 3], None)])


def test_forward_that_raises_midway():
    ops, s = drive([("root", [0, 1, 2, 3], None), ("root", [0, 1, 2, 3], 2), ("root", [0, 1, 2, 3], None)])
    assert s.pending is None and not s.active


def test_calls_outside_a_root_forward():
    ops, s = drive([("root", [0, 1, 2], None), ("direct", 1), ("direct", 1), ("root", [0, 1, 2], None), ("direct", 2)])
    assert s.pending is None


@pytest.mark.parametrize("seed", range(20))
def test_random_sequences(seed):
    rng = random.Random(seed)
    script = []
    for _ in range(8):
        if rng.random() < 0.15:
            script.append(("direct", rng.randrange(5)))
            continue
        base = list(range(5))
        if rng.random() < 0.3:
            rng.shuffle(base)
        keys = [k for k in base if rng.random() < 0.85]
        if keys and rng.random() < 0.3:
            j = rng.randrange(len(keys))
            keys.insert(j, keys[j])
        script.append(("root", keys, rng.randrange(len(keys) + 1) if keys and rng.random() < 0.2 else None))
    drive(script)


def test_run_shifted_is_declared_and_bound():
    with open(os.path.join(ROOT, "include", "zipnn_b200.h")) as f:
        h = f.read()
    args = re.search(r"int zipnn_b200_decode_plan_run_shifted\(([^)]*)\)", h)
    assert args, "zipnn_b200_decode_plan_run_shifted is not declared"
    assert len(args.group(1).split(",")) == 4
    assert "zipnn_b200_decode_plan_run_shifted" in _native.EXPORTS
