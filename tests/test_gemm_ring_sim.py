"""The shared-memory stage ring of the wgmma implicit GEMM (pcm_b200/csrc/gemm_tc.cu), replayed under
random schedules on the CPU.  One TMA producer thread and two consumer warpgroups share S stages:
full[s] (1 arrival + the TMA bytes), empty[s] (one arrival per consumer warpgroup).  A consumer
issues the wgmma group of a K block, commits it, waits until at most one group is in flight
(wgmma.wait_group 1) and only then releases the PREVIOUS block's stage; at the end of a tile it
waits for all groups and releases the last stage.  Persistent CTAs run several tiles through the
same ring.  The model checks that no TMA write lands in a stage a wgmma group has not finished
reading, that every group reads the K block it expects, and that nothing deadlocks; a variant that
releases a stage right after the commit must be caught (a self-test of the model)."""
import random

import pytest


class Bar:
    """mbarrier: `count` arrivals (plus pending TMA bytes) complete a phase."""

    def __init__(self, count):
        self.count, self.left, self.tx, self.phases = count, count, 0, 0

    def arrive(self):
        self.left -= 1
        self._maybe_flip()

    def tx_done(self):
        self.tx -= 1
        self._maybe_flip()

    def _maybe_flip(self):
        if self.left == 0 and self.tx == 0:
            self.phases += 1
            self.left = self.count

    def passed(self, parity):
        return (self.phases & 1) != parity


def simulate(rng, S, tiles, early_release=False):
    full = [Bar(1) for _ in range(S)]
    empty = [Bar(2) for _ in range(S)]
    stage_data = [None] * S          # K block (global sequence number) held by each stage
    readers = [set() for _ in range(S)]   # (consumer, group id) of wgmma groups not yet complete
    tma = []                          # in-flight TMA loads: (stage, seq)
    total = sum(tiles)

    def producer():
        stage, phase = 0, 0
        for seq in range(total):
            while not empty[stage].passed(phase ^ 1):
                yield
            if readers[stage]:
                raise AssertionError(f"TMA overwrites stage {stage} while a wgmma group still reads it")
            full[stage].tx += 1
            full[stage].arrive()
            tma.append((stage, seq))
            stage, phase = (0, phase ^ 1) if stage + 1 == S else (stage + 1, phase)

    groups = {0: [], 1: []}           # per consumer: in-order list of (gid, stage) in flight

    def consumer(c):
        stage, phase, seq, gid = 0, 0, 0, 0
        for nkb in tiles:
            prev = -1
            for _ in range(nkb):
                while not full[stage].passed(phase):
                    yield
                if stage_data[stage] != seq:
                    raise AssertionError(f"consumer {c} reads block {stage_data[stage]} instead of {seq}")
                readers[stage].add((c, gid))
                groups[c].append((gid, stage))
                gid += 1
                if early_release:
                    empty[stage].arrive()
                else:
                    while len(groups[c]) > 1:     # wgmma.wait_group 1
                        yield
                    if prev >= 0:
                        empty[prev].arrive()
                prev = stage
                seq += 1
                stage, phase = (0, phase ^ 1) if stage + 1 == S else (stage + 1, phase)
            while groups[c]:                      # wgmma.wait_group 0
                yield
            if not early_release and prev >= 0:
                empty[prev].arrive()
            yield                                 # epilogue

    actors = [producer(), consumer(0), consumer(1)]
    alive = [True, True, True]
    for _ in range(200000):
        events = [("actor", i) for i in range(3) if alive[i]]
        if tma:
            events.append(("tma", None))
        for c in (0, 1):
            if groups[c]:
                events.append(("group", c))
        if not events:
            return None
        kind, i = rng.choice(events)
        if kind == "actor":
            try:
                next(actors[i])
            except StopIteration:
                alive[i] = False
            except AssertionError as e:
                return str(e)
        elif kind == "tma":
            stage, seq = tma.pop(rng.randrange(len(tma)) if rng.random() < 0.3 else 0)
            stage_data[stage] = seq
            full[stage].tx_done()
        else:                                     # the oldest group of consumer i completes
            gid, stage = groups[i].pop(0)
            readers[stage].discard((i, gid))
    return "deadlock: no progress within the step budget"


def check(early_release, trials, seed=0):
    rng = random.Random(seed)
    for _ in range(trials):
        S = rng.choice([2, 3, 4, 8])
        tiles = [rng.randint(1, 12) for _ in range(rng.randint(1, 4))]
        bad = simulate(rng, S, tiles, early_release)
        if bad:
            return bad
    return None


def test_shipped_gemm_ring_is_clean():
    assert check(False, trials=400) is None


@pytest.mark.parametrize("seed", [1, 2])
def test_model_catches_release_before_wait(seed):
    assert check(True, trials=400, seed=seed) is not None, "the model no longer finds the known race"
