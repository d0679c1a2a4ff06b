"""DecodePipe's pinned-slab cache from many threads at once, without a GPU: pipes built and released on a loader's
threads take slabs from one process-wide cache and give them back, and no slab may be held by two of them at once."""
import sys
import threading

import torch

from zipnn_b200 import DecodePipe


def test_slab_cache_hands_each_slab_to_one_taker(monkeypatch):
    monkeypatch.setattr(DecodePipe, "_slab_cache", [])
    size = 4096
    slabs = [torch.empty(size, dtype=torch.uint8) for _ in range(8)]
    for sl in slabs:
        DecodePipe._give_slab(sl)
    DecodePipe._give_slab(torch.empty(size, dtype=torch.uint8))   # a ninth is not kept
    assert len(DecodePipe._slab_cache) == 8
    held, mu = set(), threading.Lock()
    errors = []
    barrier = threading.Barrier(8)

    def worker(i):
        try:
            barrier.wait(timeout=60)
            for _ in range(300):
                got = DecodePipe._take_slabs(size, 4)
                with mu:
                    ids = {id(sl) for sl in got}
                    assert len(ids) == len(got) and not (ids & held), "a slab handed to two takers"
                    held.update(ids)
                with mu:
                    held.difference_update(ids)
                for sl in got:
                    DecodePipe._give_slab(sl)
        except BaseException as e:   # noqa: BLE001 -- re-raised below
            errors.append(f"thread {i}: {e!r}")
            barrier.abort()

    old = sys.getswitchinterval()
    sys.setswitchinterval(1e-6)
    try:
        threads = [threading.Thread(target=worker, args=(i,)) for i in range(8)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        sys.setswitchinterval(old)
    assert not errors, errors
    assert sorted(id(s) for s in DecodePipe._slab_cache) == sorted(id(s) for s in slabs)


def test_slab_cache_drops_other_sizes(monkeypatch):
    monkeypatch.setattr(DecodePipe, "_slab_cache", [torch.empty(100, dtype=torch.uint8), torch.empty(200, dtype=torch.uint8)])
    assert [s.numel() for s in DecodePipe._take_slabs(200, 4)] == [200]
    assert DecodePipe._slab_cache == []
