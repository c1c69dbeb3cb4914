"""Executable model of a warp-specialised mbarrier pipeline with separate roles: TMA producer, MMA #1 issuer,
kEG epilogue groups, MMA #2 issuer, a scale-word ring, mbarriers with phase parity.  This was the protocol of
the tensor-core GLM kernels when they targeted tcgen05 (accumulators in tensor memory); the sm_90a kernels
use a different one, modelled in tests/test_consumer_protocol_model.py.  What stays relevant here is the
generic ring arithmetic the producer still uses (it % S, (it / S) & 1 and the arrive / parity-wait pairing of
an S-deep stage ring), exercised with many roles and barriers over thousands of schedules:

* no dead-lock for any tile count (including fewer tiles than stages / groups, partial flush periods);
* a smem stage, an eta / R buffer or a scale-ring slot is never overwritten before its consumer is done;
* every tile's eta is consumed by the group that owns the tile, with that tile's scale words;
* every tile is accumulated into G exactly once and every flush period is read out exactly once.
"""
import random

import pytest


class MBarrier:
    """mbarrier with an arrival count: the phase completes when `count` arrivals have been seen."""

    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0, "more arrivals than the barrier was initialised for"
        if self.pending == 0:
            self.pending, self.phase = self.count, self.phase ^ 1

    def passed(self, parity):  # mbarrier.try_wait.parity
        return self.phase != parity


class Pipeline:
    def __init__(self, n_it, S, kEG, kFlush, rng, threads_per_group=4):
        self.n_it, self.S, self.kEG, self.kFlush, self.rng = n_it, S, kEG, kFlush, rng
        self.ring = 2 * kEG
        T = threads_per_group  # stands for the 128 threads of an epilogue group
        self.T = T
        self.full = [MBarrier(1) for _ in range(S)]
        self.empty = [MBarrier(1) for _ in range(S)]
        self.eta_full = [MBarrier(1) for _ in range(kEG)]
        self.eta_empty = [MBarrier(T) for _ in range(kEG)]
        self.r_full = [MBarrier(T) for _ in range(kEG)]
        self.r_empty = [MBarrier(1) for _ in range(kEG)]
        self.g_full = [MBarrier(1) for _ in range(2)]
        self.g_empty = [MBarrier(T) for _ in range(2)]
        self.sf_full = [MBarrier(T) for _ in range(self.ring)]
        # data plane (what the buffers currently hold)
        self.stage = [None] * S          # tile in smem stage
        self.eta = [None] * kEG          # tile whose eta sits in TMEM buffer b
        self.r = [None] * kEG            # tile whose residuals sit in R buffer b
        self.sf = [None] * self.ring     # tile whose scale words sit in ring slot
        self.g = [[], []]                # tiles accumulated in G buffer gb since its last flush
        self.flushed = []                # (period, sorted tiles) read out by the epilogue
        self.mma2_done = set()           # tiles whose MMA #2 has completed
        self.pending_async = []          # (ready_step, callback): MMA completions / TMA arrivals
        self.step = 0

    # asynchronous engines (TMA, tensor core): complete a random number of steps later, in issue order per kind
    def later(self, fn, kind):
        last = max([t for t, _, k in self.pending_async if k == kind], default=self.step)
        self.pending_async.append((max(last, self.step + self.rng.randint(1, 6)), fn, kind))

    def producer(self):
        for it in range(self.n_it):
            st, ph = it % self.S, (it // self.S) & 1
            yield lambda: self.empty[st].passed(ph ^ 1)

            def land(it=it, st=st):
                assert self.stage[st] is None, "TMA overwrote a stage MMA #2 had not released"
                self.stage[st] = it
                self.full[st].arrive()

            self.later(land, "tma")

    def mma1(self):
        for it in range(self.n_it):
            st, ph = it % self.S, (it // self.S) & 1
            b, bph = it % self.kEG, (it // self.kEG) & 1
            slot = it % self.ring
            yield lambda: self.sf_full[slot].passed((it // self.ring) & 1)
            yield lambda: self.eta_empty[b].passed(bph ^ 1)
            yield lambda: self.full[st].passed(ph)
            assert self.stage[st] == it, "MMA #1 read a stage that does not hold its tile"
            assert self.sf[slot] == it, "MMA #1 used scale words of another tile"

            def done(it=it, b=b):
                self.eta[b] = it
                self.eta_full[b].arrive()

            self.later(done, "mma")

    def mma2(self):
        for j in range(self.n_it):
            st = j % self.S
            b, bph = j % self.kEG, (j // self.kEG) & 1
            period = j // self.kFlush
            gb = period & 1
            first = j % self.kFlush == 0
            last = j % self.kFlush == self.kFlush - 1 or j == self.n_it - 1
            slot = j % self.ring
            if first:
                yield lambda: self.g_empty[gb].passed(((period >> 1) & 1) ^ 1)
            yield lambda: self.r_full[b].passed(bph)
            assert self.r[b] == j and self.stage[st] == j and self.sf[slot] == j

            def done(j=j, st=st, b=b, gb=gb, last=last, first=first):
                if first:
                    assert self.g[gb] == [], "G buffer reused before it was flushed"
                self.g[gb].append(j)
                self.mma2_done.add(j)
                self.stage[st] = None           # stage may be refilled
                self.empty[st].arrive()
                self.r_empty[b].arrive()
                if last:
                    self.g_full[gb].arrive()

            self.later(done, "mma")

    def epilogue_thread(self, eg):
        def write_scales(t):
            slot = t % self.ring
            # the slot's previous tile must be completely consumed (by MMA #1 and MMA #2)
            prev = self.sf[slot]      # every thread of the group stores the same words for tile t
            assert prev in (None, t) or (prev == t - self.ring and prev in self.mma2_done), \
                "scale slot overwritten while in use"
            self.sf[slot] = t
            self.sf_full[slot].arrive()

        if eg < self.n_it:
            write_scales(eg)
            yield lambda: True
        for it in range(eg, self.n_it, self.kEG):
            b, bph = eg, (it // self.kEG) & 1
            yield lambda: self.eta_full[b].passed(bph)
            assert self.eta[b] == it, "epilogue group read eta of a tile it does not own"
            self.eta_empty[b].arrive()
            yield lambda: self.r_empty[b].passed(bph ^ 1)
            self.r[b] = it
            self.r_full[b].arrive()
            if it + self.kEG < self.n_it:
                yield lambda: True
                write_scales(it + self.kEG)
            last = it % self.kFlush == self.kFlush - 1 or it == self.n_it - 1
            if last:
                period = it // self.kFlush
                gb = period & 1
                yield lambda: self.g_full[gb].passed((period >> 1) & 1)
                tiles = sorted(self.g[gb])
                yield lambda: True
                self.flush_arrivals = getattr(self, "flush_arrivals", {})
                n = self.flush_arrivals.get(period, 0) + 1
                self.flush_arrivals[period] = n
                if n == self.T:                 # the last thread of the group finishes the read-out
                    self.flushed.append((period, tiles))
                    self.g[gb] = []
                self.g_empty[gb].arrive()

    def run(self):
        actors = [self.producer(), self.mma1(), self.mma2()]
        actors += [self.epilogue_thread(eg) for eg in range(self.kEG) for _ in range(self.T)]
        waiting = [None] * len(actors)   # predicate an actor is blocked on
        alive = [True] * len(actors)
        for i, a in enumerate(actors):
            try:
                waiting[i] = next(a)
            except StopIteration:
                alive[i] = False
        limit = 400 * (self.n_it + 4) * len(actors)
        while any(alive) or self.pending_async:
            self.step += 1
            assert self.step < limit, "live-lock"
            due = [p for p in self.pending_async if p[0] <= self.step]
            for p in sorted(due, key=lambda p: p[0]):
                self.pending_async.remove(p)
                p[1]()
            runnable = [i for i in range(len(actors)) if alive[i] and waiting[i]()]
            if not runnable:
                assert self.pending_async, f"dead-lock at step {self.step}"
                self.step = min(p[0] for p in self.pending_async) - 1
                continue
            i = self.rng.choice(runnable)
            try:
                waiting[i] = next(actors[i])
            except StopIteration:
                alive[i] = False
        return self


@pytest.mark.parametrize("kEG", [1, 2, 3, 4])
def test_pipeline_protocol_has_no_deadlock_and_no_buffer_reuse(kEG):
    rng = random.Random(1234 + kEG)
    for trial in range(150):
        n_it = rng.choice([0, 1, 2, 3, 4, 5, 7, 8, 9, 13, 16, 17, 31, 40])
        S = rng.randint(2, 6)
        kFlush = rng.choice([2, 4, 8])
        p = Pipeline(n_it, S, kEG, kFlush, random.Random(rng.random())).run()
        periods = (n_it + kFlush - 1) // kFlush
        assert [f[0] for f in sorted(p.flushed)] == list(range(periods)), (n_it, S, kEG, kFlush)
        seen = [t for _, tiles in sorted(p.flushed) for t in tiles]
        assert seen == list(range(n_it)), "every tile must be accumulated and flushed exactly once"
        for period, tiles in p.flushed:
            assert tiles == list(range(period * kFlush, min(n_it, (period + 1) * kFlush)))


def test_model_detects_a_broken_protocol():
    """Sanity of the checker itself: a scale ring that is too shallow (kEG slots instead of 2 kEG) lets the
    epilogue overwrite words MMA #2 still needs — the model must notice."""

    class Shallow(Pipeline):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.ring = self.kEG
            self.sf = [None] * self.ring
            self.sf_full = [MBarrier(self.T) for _ in range(self.ring)]

    rng = random.Random(7)
    with pytest.raises(AssertionError):
        for _ in range(50):
            Shallow(24, 4, 2, 4, random.Random(rng.random())).run()
