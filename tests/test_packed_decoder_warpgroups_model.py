"""Executable model of the bf16 tensor-core GLM kernel's 512-thread layout (csrc/glm_tc.cu, "Packed X"): warp 0 is the
producer, warps 1 to 3 (warpgroup 0) and 12 to 15 (warpgroup 3) decode the packed X, warpgroups 1 and 2 consume.
The 224 decoder threads are one team: the kXBlock chunks of every panel are strided over all of them (thread td
decodes chunks td, td + 224, ...: 5 for td < 128, 4 for the rest), every thread reads every compressed slot it
waits for and releases it after its stores (xempty counts 224), the row data and the exceptions are spread over all
224, and a stage is full once all 224 have arrived.  Around the roles, setmaxnreg moves registers per warpgroup: the
consumer warpgroups go from 128 to 168 per thread and back, warpgroups 0 and 3 from 128 to 88 and back, then every
thread meets at the CTA's __syncthreads.  An inc blocks until the CTA's pool holds the registers.

A randomised scheduler interleaves the threads; the model checks, for every interleaving:

* no dead-lock, for packed and bf16 launches (where the decoders only move their registers), any chunk table, slot
  count, panel count and load group, with the register moves and the shared tail included;
* a compressed slot is refilled only after every thread that read it has released it, and a decoder reads a slot
  only once it holds the panel it expects;
* a stage is decoded into only after every consumer thread has released it, and consumed only once every decoder has
  stored all of its chunks of every panel and the exceptions are patched; every chunk of a tile is written once;
* the register pool never goes negative and every warpgroup is back at 128 at the shared tail; without barrier 3, an
  idle warpgroup that takes its registers back at once starves a consumer warpgroup (a dead-lock the model finds);
* with pipeline stalls injected, every thread still leaves its loop and reaches the tail.

D_A / D_B decoder threads and C chunks per panel stand for 96 / 128 and 1024; index / parity formulas are the
kernel's (it % S, (it / S) & 1, x % X, (x / X) & 1, j % kRing).  A change to the kernel's protocol has to be mirrored
here.
"""
import random

import pytest

from test_consumer_protocol_model import MBarrier, NamedBarrier

REGS, CONSUMER_REGS, OTHER_REGS = 128, 168, 88


def chunks_of(td, D, C):
    """The chunks of a panel that decoder thread td decodes (the kernel's i = td + k * kDecThreads, i < 1024)."""
    return list(range(td, C, D))


class RegisterPool:
    """setmaxnreg per warpgroup: every thread of the warpgroup arrives, then the warpgroup's count changes; dec returns
    registers to the CTA's pool at once, inc waits until the pool holds them.  Every warpgroup of the kernel has 128
    threads, so the pool counts registers per thread of a warpgroup, whatever threads the model runs for it."""

    def __init__(self, sizes):
        self.free = 0
        self.regs = [REGS] * len(sizes)
        self.sizes = sizes
        self.arrived = [0] * len(sizes)
        self.gen = [0] * len(sizes)
        self.want = [None] * len(sizes)

    def set(self, wg, n):
        g = self.gen[wg]
        self.arrived[wg] += 1
        if self.arrived[wg] == self.sizes[wg]:   # the warpgroup's instruction issues once all of its threads are there
            self.arrived[wg] = 0
            self.want[wg] = n
        # ready once the change went through, or once the pool can serve it (dec: always; inc: setmaxnreg.inc blocks
        # until the pool holds the registers); the thread the scheduler runs first then makes it
        yield lambda: self.gen[wg] != g or (self.want[wg] is not None and self.free >= self.want[wg] - self.regs[wg])
        if self.gen[wg] == g:
            self.free -= self.want[wg] - self.regs[wg]
            assert self.free >= 0
            self.regs[wg], self.want[wg], self.gen[wg] = self.want[wg], None, g + 1


def run(chunks, X, panels, group, seed, pk=True, D_A=3, D_B=4, C=9, T=2, n_ex=3, fault_prob=0.0, kRing=8, preload=0,
        hand_back_barrier=True):
    """chunks: tile counts; X compressed slots, 2 stages; group: panels per load group; D_A + D_B decoder threads in
    warpgroups 0 and 3, C chunks per panel, T threads per consumer warpgroup; n_ex exceptions per tile;
    hand_back_barrier: warpgroups 0 and 3 take their registers back only after barrier 3, which the consumers reach
    once they have returned theirs (the kernel's order; False drops the barrier)."""
    rng = random.Random(seed)
    S, D = 2, D_A + D_B
    fault = [False]
    ng = group if panels % group == 0 and X >= group else 1
    full = [MBarrier(D if pk else 1) for _ in range(S)]
    empty = [MBarrier(2 * T) for _ in range(S)]
    xfull = [MBarrier(1) for _ in range(X)]
    xempty = [MBarrier(D) for _ in range(X)]
    bar_ring = [MBarrier(1) for _ in range(kRing)]
    ring = [None] * kRing
    slot = [None] * X
    readers = [set() for _ in range(X)]   # decoder threads that read the slot's current panel and have not released it
    stage = [[[None] * C for _ in range(panels)] for _ in range(S)]
    patched = [None] * S
    writes = {}
    bar1, bar2 = NamedBarrier(2 * T), NamedBarrier(D)
    sizes = [1 + D_A, T, T, D_B]          # threads per warpgroup: 0 = producer + decoders A, 1 and 2 consumers, 3 decoders B
    pool = RegisterPool(sizes)
    tail = NamedBarrier(sum(sizes))       # __syncthreads before the CTA's fold
    bar3 = NamedBarrier(sum(sizes))       # the consumers have returned their registers
    decided1, decided2 = [None], [None]
    consumed, at_tail = {}, []

    def mbar_wait(bar, parity):
        yield lambda: bar.passed(parity) or fault[0]

    # early loads: up to every compressed slot (packed), or every stage but the one theta is staged in (bf16)
    preloaded = min(preload, chunks[0] * panels if pk else min(chunks[0], S - 1)) if chunks else 0
    loads = [(t, p) for t in range(sum(chunks)) for p in range(panels)]

    def take_back(wg):          # warpgroups 0 and 3, after their roles
        if hand_back_barrier:
            yield from bar3.sync()
        yield from pool.set(wg, REGS)

    def give_back(wg):          # the consumer warpgroups, after theirs
        yield from pool.set(wg, REGS)
        if hand_back_barrier:
            yield from bar3.sync()

    def shared_tail(wg):
        at_tail.append(pool.regs[wg])
        yield from tail.sync()

    def producer():
        yield from pool.set(0, OTHER_REGS)
        x, it = 0, 0
        for j in range(len(chunks) + 1):
            ch = chunks[j] if j < len(chunks) else -1
            ring[j % kRing] = ch
            bar_ring[j % kRing].arrive()
            if ch < 0:
                break
            for _ in range(ch * panels if pk else 0):
                if not (j == 0 and x < preloaded):
                    yield from mbar_wait(xempty[x % X], ((x // X) & 1) ^ 1)
                    if not fault[0]:
                        assert not readers[x % X], "slot refilled before every thread that read it released it"
                    slot[x % X] = loads[x]
                    xfull[x % X].arrive()
                x += 1
            for _ in range(0 if pk else ch):   # bf16: the producer fills the stage itself (full counts 1)
                s = it % S
                if not (j == 0 and it < preloaded):
                    yield from mbar_wait(empty[s], ((it // S) & 1) ^ 1)
                    for p in range(panels):
                        stage[s][p] = [it] * C
                    patched[s] = it
                    full[s].arrive()
                it += 1
        yield from take_back(0)
        yield from shared_tail(0)

    def early_loads():
        for x in range(preloaded):
            if pk:
                slot[x] = loads[x]
                xfull[x].arrive()
            else:
                for p in range(panels):
                    stage[x][p] = [x] * C
                patched[x] = x
                full[x].arrive()

    def decoder(td):
        wg = 0 if td < D_A else 3
        yield from pool.set(wg, OTHER_REGS)
        it, x, j = 0, 0, 0
        while pk:
            yield from mbar_wait(bar_ring[j % kRing], (j // kRing) & 1)
            yield from bar2.sync()
            if td == 0:
                decided2[0] = -1 if fault[0] else ring[j % kRing]
            yield from bar2.sync()
            ch = decided2[0]
            if ch < 0:
                break
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
                            readers[x % X].add(td)
                        held.append(x % X)
                        x += 1
                    for h in range(ng):   # decode and store this thread's chunks of each panel, then release its slot
                        yield lambda: True
                        for i in chunks_of(td, D, C):
                            stage[s][p0 + h][i] = it
                            if not fault[0]:
                                writes[(it, p0 + h, i)] = writes.get((it, p0 + h, i), 0) + 1
                        readers[held[h]].discard(td)
                        xempty[held[h]].arrive()
                yield from bar2.sync()    # the exceptions are patched once every thread's stores are in
                if not fault[0]:
                    assert all(stage[s][p] == [it] * C for p in range(panels)), "exception patched before every store"
                for e in range(td, n_ex, D):
                    yield lambda: True
                if td == 0:
                    patched[s] = it
                full[s].arrive()
                it += 1
            j += 1
        yield from take_back(wg)
        yield from shared_tail(wg)

    def consumer(wg, tid):
        yield from pool.set(wg, CONSUMER_REGS)
        it, j = 0, 0
        while True:
            yield from mbar_wait(bar_ring[j % kRing], (j // kRing) & 1)
            yield from bar1.sync()
            if wg == 1 and tid == 0:
                decided1[0] = -1 if fault[0] else ring[j % kRing]
            yield from bar1.sync()
            ch = decided1[0]
            if ch < 0:
                break
            for _ in range(ch):
                s = it % S
                yield from mbar_wait(full[s], (it // S) & 1)
                if not fault[0]:
                    assert all(stage[s][p] == [it] * C for p in range(panels)) and patched[s] == it, \
                        "stage consumed before every decoder stored it"
                yield from bar1.sync()
                if not fault[0]:
                    assert all(stage[s][p] == [it] * C for p in range(panels)), "stage rewritten while it was consumed"
                    consumed[(wg, tid, it)] = consumed.get((wg, tid, it), 0) + 1
                empty[s].arrive()
                it += 1
            j += 1
        yield from give_back(wg)
        yield from shared_tail(wg)

    early_loads()
    roles = ([producer()] + [decoder(td) for td in range(D)]
             + [consumer(wg, t) for wg in (1, 2) for t in range(T)])
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
    assert at_tail == [REGS] * len(roles), "a warpgroup reached the shared tail with a changed register count"
    assert pool.free == 0 and pool.regs == [REGS] * 4
    return writes, consumed, fault[0]


def test_the_decoder_split_covers_a_panel_once():
    # the kernel's numbers: 1024 chunks of a panel over 224 threads, 5 chunks for the first 128, 4 for the rest
    per = [chunks_of(td, 224, 1024) for td in range(224)]
    assert sorted(i for p in per for i in p) == list(range(1024))
    assert [len(p) for p in per] == [5] * 128 + [4] * 96
    assert 256 * CONSUMER_REGS + 256 * OTHER_REGS == 65536 == 512 * REGS


@pytest.mark.parametrize("X,panels,group,preload", [(6, 4, 2, 6), (6, 4, 1, 6), (2, 4, 2, 2), (2, 2, 1, 0),
                                                    (3, 4, 2, 3), (5, 2, 2, 5)])
@pytest.mark.parametrize("chunks", [[2], [2, 2], [32, 4, 4], [4, 6, 2, 2]])
def test_every_chunk_is_decoded_once_and_every_tile_consumed_once(chunks, X, panels, group, preload):
    D, C, T = 7, 9, 2
    for seed in range(4):
        writes, consumed, faulted = run(chunks, X, panels, group, seed, C=C, T=T, preload=preload)
        assert not faulted
        n = sum(chunks)
        assert writes == {(it, p, i): 1 for it in range(n) for p in range(panels) for i in range(C)}
        assert consumed == {(wg, t, it): 1 for wg in (1, 2) for t in range(T) for it in range(n)}


@pytest.mark.parametrize("chunks", [[2], [32, 4, 4], [4, 6, 2, 2]])
def test_a_bf16_launch_moves_the_idle_decoders_registers_and_ends(chunks):
    for seed in range(6):
        writes, consumed, faulted = run(chunks, 6, 4, 2, seed, pk=False, preload=1)
        assert not faulted and not writes
        assert consumed == {(wg, t, it): 1 for wg in (1, 2) for t in range(2) for it in range(sum(chunks))}


@pytest.mark.parametrize("pk", [True, False])
@pytest.mark.parametrize("X,panels,group,preload", [(6, 4, 2, 6), (2, 4, 2, 0), (4, 2, 1, 4)])
@pytest.mark.parametrize("chunks", [[2, 2], [32, 4, 4], [4, 6, 2, 2]])
def test_a_stalled_pipeline_never_leaves_a_thread_waiting(chunks, X, panels, group, preload, pk):
    for seed in range(40):
        run(chunks, X, panels, group, seed, pk=pk, fault_prob=0.01, preload=preload)   # terminates: asserted in run()


def test_idle_warpgroups_taking_registers_back_early_would_dead_lock():
    # a bf16 launch: the decoders have no work and, without barrier 3, take their registers back before a consumer
    # warpgroup got its own; some interleaving then leaves that warpgroup, and the other at barrier 1, waiting
    hung = 0
    for seed in range(40):
        try:
            run([2, 2], 6, 4, 2, seed, pk=False, hand_back_barrier=False)
        except AssertionError as ex:
            assert "dead-lock" in str(ex) or "did not terminate" in str(ex)
            hung += 1
    assert hung > 0
