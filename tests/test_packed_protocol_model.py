"""Executable model of the packed-X pipeline of the bf16 tensor-core GLM kernel (csrc/glm_tc.cu, "Packed X"): the
producer (warp 0) streams compressed panels into a ring of slots, the decoders (warps 1 to 3, named barrier 2) decode
each tile's panels into a bf16 stage and arrive on its `full` barrier (one arrival per decoder thread), and the two
consumer warpgroups (named barrier 1) use the stage as in tests/test_consumer_protocol_model.py.  A randomised
scheduler interleaves the threads; the model checks, for every interleaving:

* no dead-lock for any chunk table, slot count and panel count (fewer slots than panels included);
* a compressed slot is refilled only after every decoder thread has released it, and a decoder reads a slot only
  once it holds the panel it expects;
* a bf16 stage is decoded into only after every consumer thread has released it, and consumed only once every
  decoder thread has written its part of it (this tile's);
* a decoder reads the tile's footer after every decoder has copied its part, and the footer buffer of a tile is not
  overwritten (two tiles later) while a decoder still patches from it;
* every tile is decoded once by every decoder thread and consumed once by every consumer thread;
* with pipeline stalls injected, every thread still leaves its loop: decoders and consumers each decide a chunk
  together (barrier, one thread reads the fault flag and the ring entry, barrier).

Index / parity formulas are the kernel's (it % S, (it / S) & 1, x % X, (x / X) & 1, j % kRing); a change to the
kernel's protocol has to be mirrored here.
"""
import random

import pytest

from test_consumer_protocol_model import MBarrier, NamedBarrier


def run(chunks, S, X, panels, seed, D=3, T=2, fault_prob=0.0, kRing=8, preload=0):
    """chunks: tile counts; S bf16 stages, X compressed slots; D decoder threads (stand for 96), T threads per
    consumer warpgroup (stand for 128); preload: panel loads issued before any other role runs (early loads)."""
    rng = random.Random(seed)
    fault = [False]
    full = [MBarrier(D) for _ in range(S)]
    empty = [MBarrier(2 * T) for _ in range(S)]
    xfull = [MBarrier(1) for _ in range(X)]
    xempty = [MBarrier(D) for _ in range(X)]
    bar_ring = [MBarrier(1) for _ in range(kRing)]
    ring = [None] * kRing
    slot = [None] * X
    stage = [[None] * D for _ in range(S)]
    foot = [[None] * D for _ in range(2)]
    bar1, bar2 = NamedBarrier(2 * T), NamedBarrier(D)
    decided1, decided2 = [None], [None]
    decoded, consumed = {}, {}

    def mbar_wait(bar, parity):
        yield lambda: bar.passed(parity) or fault[0]

    # the kernel's `preloaded`: the first chunk's panels, at most one per slot
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
                if not (j == 0 and x < preloaded):   # else issued before theta arrived, into a fresh slot
                    yield from mbar_wait(xempty[x % X], ((x // X) & 1) ^ 1)
                    if not fault[0]:
                        assert xempty[x % X].pending == D, "slot refilled before every decoder released it"
                    slot[x % X] = loads[x]
                    xfull[x % X].arrive()
                x += 1

    def early_loads():   # the producer's loads before the prologue: slots 0 .. preloaded - 1 are fresh
        for x in range(preloaded):
            slot[x] = loads[x]
            xfull[x].arrive()

    def decoder(tid):
        it, x, j, fb = 0, 0, 0, 0
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
                yield from mbar_wait(empty[it % S], ((it // S) & 1) ^ 1)
                if not fault[0]:
                    assert empty[it % S].pending == 2 * T, "stage decoded into before every consumer released it"
                for p in range(panels):
                    yield from mbar_wait(xfull[x % X], (x // X) & 1)
                    if not fault[0]:
                        assert slot[x % X] == (it, p), "decoder read a slot that does not hold its panel"
                    if p == 0:
                        foot[fb][tid] = it
                    stage[it % S][tid] = it
                    xempty[x % X].arrive()
                    x += 1
                yield from bar2.sync()
                yield lambda: True   # the patch step: other threads may run ahead in between
                if not fault[0]:
                    assert foot[fb] == [it] * D, "footer patched from before every decoder copied it, or overwritten"
                    decoded[(tid, it)] = decoded.get((tid, it), 0) + 1
                full[it % S].arrive()
                it += 1
                fb ^= 1
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
                yield from mbar_wait(full[it % S], (it // S) & 1)
                if not fault[0]:
                    assert stage[it % S] == [it] * D, "stage consumed before every decoder wrote this tile"
                yield from bar1.sync()
                if not fault[0]:
                    assert stage[it % S] == [it] * D, "stage rewritten while it was consumed"
                    consumed[(wg, tid, it)] = consumed.get((wg, tid, it), 0) + 1
                empty[it % S].arrive()
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


@pytest.mark.parametrize("S,X,panels,preload", [(2, 6, 4, 6), (2, 3, 4, 0), (2, 2, 2, 2), (2, 5, 2, 5), (3, 2, 4, 2)])
@pytest.mark.parametrize("chunks", [[2], [2, 2], [32, 4, 4], [4, 6, 2, 2], [4] * 8])
def test_every_tile_is_decoded_and_consumed_once(chunks, S, X, panels, preload):
    D, T = 3, 2
    for seed in range(8):
        decoded, consumed, faulted = run(chunks, S, X, panels, seed, D=D, T=T, preload=preload)
        assert not faulted
        n = sum(chunks)
        assert decoded == {(t, it): 1 for t in range(D) for it in range(n)}
        assert consumed == {(wg, t, it): 1 for wg in range(2) for t in range(T) for it in range(n)}


@pytest.mark.parametrize("S,X,panels,preload", [(2, 6, 4, 6), (2, 2, 2, 0)])
@pytest.mark.parametrize("chunks", [[2, 2], [32, 4, 4], [4, 6, 2, 2]])
def test_a_stalled_packed_pipeline_never_leaves_a_thread_waiting(chunks, S, X, panels, preload):
    for seed in range(60):
        run(chunks, S, X, panels, seed, fault_prob=0.01, preload=preload)   # terminates: asserted inside run()
