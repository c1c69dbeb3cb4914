"""Executable model of the packed-X decoders of the bf16 tensor-core GLM kernel (csrc/glm_tc.cu, "Packed X") when they
decode a tile's panels in groups: each decoder thread (warps 1 to 3) waits for the compressed slots of the group's ng
panels one after the other, loads its part of each into registers, then decodes and stores the panels in order and
releases each slot after its panel's stores.  A group holds ng slots at once.  The kernel's groups hold 2 panels
(1 in the instantiations whose registers do not allow 2: the per-panel protocol of tests/test_packed_protocol_model.py);
every packed launch has at least 2 slots and 2 or 4 panels, so a group always fits and divides the tile.  The model
also runs larger groups, and shows that a group needs no more slots than the ring has.  A randomised scheduler
interleaves the threads; the model checks, for every interleaving:

* no dead-lock for any chunk table, slot count, panel count and group size the kernel allows (ng = X included);
* a compressed slot is refilled only after every decoder thread has released it, and a decoder reads a slot only once
  it holds the panel it expects;
* a bf16 stage is decoded into only after every consumer thread has released it, and consumed only once every decoder
  thread has written all of its panels (this tile's);
* every tile is decoded once by every decoder thread and consumed once by every consumer thread;
* with pipeline stalls injected, every thread still leaves its loop.

Index / parity formulas are the kernel's (it % S, (it / S) & 1, x % X, (x / X) & 1, j % kRing); a change to the
kernel's protocol has to be mirrored here.
"""
import random

import pytest

from test_consumer_protocol_model import MBarrier, NamedBarrier


def group_size(group, panels, X):
    """Panels per group: ``group`` where it divides the panels and fits in the slots (always so for the kernel's groups
    of 2), else 1."""
    return group if panels % group == 0 and X >= group else 1


def run(chunks, S, X, panels, group, seed, D=3, T=2, fault_prob=0.0, kRing=8, preload=0):
    """chunks: tile counts; S bf16 stages, X compressed slots; group: the instantiation's panels per load group; D
    decoder threads (stand for 96), T threads per consumer warpgroup (stand for 128); preload: panel loads issued
    before any other role runs (early loads)."""
    rng = random.Random(seed)
    fault = [False]
    ng = group_size(group, panels, X)
    full = [MBarrier(D) for _ in range(S)]
    empty = [MBarrier(2 * T) for _ in range(S)]
    xfull = [MBarrier(1) for _ in range(X)]
    xempty = [MBarrier(D) for _ in range(X)]
    bar_ring = [MBarrier(1) for _ in range(kRing)]
    ring = [None] * kRing
    slot = [None] * X
    stage = [[[None] * D for _ in range(panels)] for _ in range(S)]
    bar1, bar2 = NamedBarrier(2 * T), NamedBarrier(D)
    decided1, decided2 = [None], [None]
    decoded, consumed = {}, {}

    def mbar_wait(bar, parity):
        yield lambda: bar.passed(parity) or fault[0]

    preloaded = min(preload, chunks[0] * panels) if chunks else 0
    loads = [(t, p) for t in range(sum(chunks)) for p in range(panels)]

    def producer():
        x = 0
        for j in range(len(chunks) + 1):
            ch = chunks[j] if j < len(chunks) else -1
            ring[j % kRing] = ch
            bar_ring[j % kRing].arrive()
            if ch < 0:
                return
            for _ in range(ch * panels):
                if not (j == 0 and x < preloaded):
                    yield from mbar_wait(xempty[x % X], ((x // X) & 1) ^ 1)
                    if not fault[0]:
                        assert xempty[x % X].pending == D, "slot refilled before every decoder released it"
                    slot[x % X] = loads[x]
                    xfull[x % X].arrive()
                x += 1

    def early_loads():
        for x in range(preloaded):
            slot[x] = loads[x]
            xfull[x].arrive()

    def decoder(tid):
        it, x, j = 0, 0, 0
        while True:
            yield from mbar_wait(bar_ring[j % kRing], (j // kRing) & 1)
            yield from bar2.sync()
            if tid == 0:
                decided2[0] = -1 if fault[0] else ring[j % kRing]
            yield from bar2.sync()
            ch = decided2[0]
            if ch < 0:
                return
            for _ in range(ch):
                s = it % S
                yield from mbar_wait(empty[s], ((it // S) & 1) ^ 1)
                if not fault[0]:
                    assert empty[s].pending == 2 * T, "stage decoded into before every consumer released it"
                for p0 in range(0, panels, ng):
                    held = []
                    for h in range(ng):   # the group's loads: every slot waited for, none released yet
                        yield from mbar_wait(xfull[x % X], (x // X) & 1)
                        if not fault[0]:
                            assert slot[x % X] == (it, p0 + h), "decoder read a slot that does not hold its panel"
                        held.append(x % X)
                        x += 1
                    for h in range(ng):   # decode and store each panel, then release its slot
                        yield lambda: True
                        stage[s][p0 + h][tid] = it
                        xempty[held[h]].arrive()
                yield from bar2.sync()    # the exceptions are patched once every thread's stores are in
                if not fault[0]:
                    decoded[(tid, it)] = decoded.get((tid, it), 0) + 1
                full[s].arrive()
                it += 1
            j += 1

    def consumer(wg, tid):
        it, j = 0, 0
        while True:
            yield from mbar_wait(bar_ring[j % kRing], (j // kRing) & 1)
            yield from bar1.sync()
            if wg == 0 and tid == 0:
                decided1[0] = -1 if fault[0] else ring[j % kRing]
            yield from bar1.sync()
            ch = decided1[0]
            if ch < 0:
                return
            for _ in range(ch):
                s = it % S
                yield from mbar_wait(full[s], (it // S) & 1)
                if not fault[0]:
                    assert all(stage[s][p] == [it] * D for p in range(panels)), "stage consumed before it was decoded"
                yield from bar1.sync()
                if not fault[0]:
                    assert all(stage[s][p] == [it] * D for p in range(panels)), "stage rewritten while it was consumed"
                    consumed[(wg, tid, it)] = consumed.get((wg, tid, it), 0) + 1
                empty[s].arrive()
                it += 1
            j += 1

    early_loads()
    roles = [producer()] + [decoder(t) for t in range(D)] + [consumer(wg, t) for wg in range(2) for t in range(T)]
    waiting = [next(r, None) for r in roles]
    for _ in range(400000):
        live = [i for i, w in enumerate(waiting) if w is not None]
        if not live:
            break
        if fault_prob and not fault[0] and rng.random() < fault_prob:
            fault[0] = True   # a bounded wait somewhere gave up
        ready = [i for i in live if waiting[i]()]
        if not ready:
            assert fault_prob and not fault[0], "dead-lock"
            fault[0] = True   # every blocked mbarrier wait times out eventually
            continue
        i = rng.choice(ready)
        waiting[i] = next(roles[i], None)
    else:
        raise AssertionError("did not terminate")
    return decoded, consumed, fault[0]


@pytest.mark.parametrize("X,panels,group,preload", [(6, 4, 2, 6), (6, 4, 4, 6), (4, 4, 4, 0), (2, 4, 2, 2),
                                                    (2, 2, 2, 0), (3, 4, 4, 3), (2, 4, 4, 2), (5, 2, 4, 5)])
@pytest.mark.parametrize("chunks", [[2], [2, 2], [32, 4, 4], [4, 6, 2, 2], [4] * 8])
def test_every_tile_is_decoded_and_consumed_once_in_groups(chunks, X, panels, group, preload):
    D, T = 3, 2
    for seed in range(6):
        decoded, consumed, faulted = run(chunks, 2, X, panels, group, seed, D=D, T=T, preload=preload)
        assert not faulted
        n = sum(chunks)
        assert decoded == {(t, it): 1 for t in range(D) for it in range(n)}
        assert consumed == {(wg, t, it): 1 for wg in range(2) for t in range(T) for it in range(n)}


def test_a_group_never_holds_more_slots_than_there_are():
    assert group_size(4, 4, 3) == 1 and group_size(4, 2, 6) == 1 and group_size(2, 4, 2) == 2


@pytest.mark.parametrize("X,panels,group,preload", [(6, 4, 4, 6), (2, 4, 2, 0), (4, 4, 4, 4)])
@pytest.mark.parametrize("chunks", [[2, 2], [32, 4, 4], [4, 6, 2, 2]])
def test_a_stalled_grouped_pipeline_never_leaves_a_thread_waiting(chunks, X, panels, group, preload):
    for seed in range(60):
        run(chunks, 2, X, panels, group, seed, fault_prob=0.01, preload=preload)   # terminates: asserted inside run()
