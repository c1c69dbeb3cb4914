"""Executable model of the sm_90a tensor-core GLM pipeline (csrc/glm_tc.cu, csrc/glm_fp8.cu): one TMA producer,
two consumer warpgroups that share every tile and meet at named barrier 1 (256 threads), mbarriers with phase
parity.  A randomised scheduler interleaves the threads; the model checks, for every interleaving:

* no dead-lock for any chunk table (fewer tiles than stages, one-tile chunks, many chunks);
* an X stage is refilled only after every consumer thread has arrived on its `empty` barrier (256 arrivals);
* the residual buffer R[it % 2] written before the per-tile barrier holds the rows of THIS tile from both
  warpgroups when the gradient MMA reads it, and is not rewritten while the other warpgroup still reads it;
* every tile is consumed exactly once by every consumer thread;
* with pipeline stalls injected (a bounded mbarrier wait gives up and raises the CTA's fault flag at a random
  moment), every thread still leaves its loop: the consumers decide each chunk together (barrier, one thread
  reads the flag and the ring entry, barrier), so no warpgroup is left waiting at a named barrier.

Index / parity formulas are the kernel's (it % S, (it / S) & 1, j % kRing, (j / kRing) & 1); a change to the
kernels' protocol has to be mirrored here.
"""
import random

import pytest


class MBarrier:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0, "more arrivals than the barrier was initialised for"
        if self.pending == 0:
            self.pending, self.phase = self.count, self.phase ^ 1

    def passed(self, parity):  # mbarrier.try_wait.parity
        return self.phase != parity


class NamedBarrier:
    """bar.sync id, count: hardware counts arrivals, whatever program point they come from."""

    def __init__(self, count):
        self.count, self.arrived, self.gen = count, 0, 0

    def sync(self):
        g = self.gen
        self.arrived += 1
        if self.arrived == self.count:
            self.arrived, self.gen = 0, self.gen + 1
        yield lambda: self.gen != g


def run(chunks, S, T, seed, fault_prob=0.0, kRing=8):
    """chunks: tile counts; T threads per consumer warpgroup (stands for 128)."""
    rng = random.Random(seed)
    fault = [False]
    full = [MBarrier(1) for _ in range(S)]
    empty = [MBarrier(2 * T) for _ in range(S)]
    bar_ring = [MBarrier(1) for _ in range(kRing)]
    ring = [None] * kRing
    stage = [None] * S
    R = [[None, None] for _ in range(2)]
    bar1 = NamedBarrier(2 * T)
    decided = [None]
    consumed = {}

    def mbar_wait(bar, parity):
        yield lambda: bar.passed(parity) or fault[0]

    def producer():
        it = 0
        for j in range(len(chunks) + 1):
            ch = chunks[j] if j < len(chunks) else -1
            ring[j % kRing] = ch
            bar_ring[j % kRing].arrive()
            if ch < 0:
                return
            for _ in range(ch):
                yield from mbar_wait(empty[it % S], ((it // S) & 1) ^ 1)
                if not fault[0]:
                    assert empty[it % S].pending == 2 * T, "stage refilled before every consumer released it"
                stage[it % S] = it
                full[it % S].arrive()
                it += 1

    def consumer(wg, tid):
        it, j = 0, 0
        while True:
            slot = j % kRing
            yield from mbar_wait(bar_ring[slot], (j // kRing) & 1)
            yield from bar1.sync()
            if wg == 0 and tid == 0:
                decided[0] = -1 if fault[0] else ring[slot]
            yield from bar1.sync()
            ch = decided[0]
            if ch < 0:
                return
            for _ in range(ch):
                yield from mbar_wait(full[it % S], (it // S) & 1)
                if not fault[0]:
                    assert stage[it % S] == it
                R[it % 2][wg] = it
                yield from bar1.sync()
                if not fault[0]:
                    assert R[it % 2] == [it, it], "R read before both warpgroups wrote this tile's rows"
                    assert stage[it % S] == it
                    consumed[(wg, tid, it)] = consumed.get((wg, tid, it), 0) + 1
                empty[it % S].arrive()
                it += 1
            j += 1

    roles = [producer()] + [consumer(wg, t) for wg in range(2) for t in range(T)]
    waiting = [next(r, None) for r in roles]
    for _ in range(200000):
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
    return consumed, fault[0]


@pytest.mark.parametrize("S", [2, 3, 4])
@pytest.mark.parametrize("chunks", [[1], [2, 2], [32, 4, 4], [1, 3, 1, 5, 2, 2, 7], [4] * 12])
def test_every_tile_is_consumed_once_by_every_thread(chunks, S):
    T = 3
    for seed in range(20):
        consumed, faulted = run(chunks, S, T, seed)
        assert not faulted
        n = sum(chunks)
        assert consumed == {(wg, t, it): 1 for wg in range(2) for t in range(T) for it in range(n)}


@pytest.mark.parametrize("S", [2, 4])
@pytest.mark.parametrize("chunks", [[2, 2], [32, 4, 4], [1, 3, 1, 5, 2, 2, 7]])
def test_a_stalled_pipeline_never_leaves_a_thread_waiting(chunks, S):
    for seed in range(200):
        run(chunks, S, 3, seed, fault_prob=0.02)   # terminates: asserted inside run()
