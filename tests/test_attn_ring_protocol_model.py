"""Model check (CPU) of the synchronisation protocol of csrc/attn.cu — one TMA producer warp, a kStages-deep K/V^T ring, two
consumer warpgroups that each read every key tile.

The kernel cannot be run here (no GPU), so its wait graph is restated as a small discrete-event model: mbarriers with phase
parity exactly as `mbarrier.try_wait.parity` sees them (a wait on parity P passes iff the barrier's current phase has the other
parity — so a waiter that is overtaken by two completions would pass on a stale phase, which is the aliasing hazard to rule out),
one agent per role (producer, each consumer warpgroup, the TMA engine that lands issued loads in any order, and for the fused
sequence-parallel gather the copy engine that raises one flag per K/V segment), random interleavings.  Checked:
  * no deadlock (every agent terminates),
  * a consumer reads tile j only after its bytes landed, and finds tile j (not an older or newer one) in the slot, also after
    its MMAs (the slot is not refilled under them),
  * the producer refills slot j % kStages with tile j + kStages only after BOTH warpgroups released tile j (kv_empty counts 2),
  * with segment flags, a tile is loaded only after the flag of its segment was seen.
The statements mirror the code: kv_full parity (j / kStages) & 1, kv_empty parity ((j / kStages) & 1) ^ 1, q_full parity 0,
one kv_empty arrival per consumer warpgroup per tile, `ready_seg` caching the last segment whose flag was seen."""
import random

import pytest


class MBar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0      # phase = number of completed phases

    def arrive(self):
        self.pending -= 1
        if self.pending == 0:
            self.pending, self.phase = self.count, self.phase + 1

    def passed(self, parity):                                         # try_wait.parity semantics
        return (self.phase & 1) != parity


class Aliasing(AssertionError):
    pass


class Deadlock(AssertionError):
    pass


def simulate(n_kv, rng, stages=6, n_cons=2, empty_count=None, segs=None, producer_parity_bug=False):
    """Runs one random schedule; returns the event log.  segs: key tiles per K/V segment (fused gather; None = no flags).
    empty_count / producer_parity_bug: deliberately wrong variants the checks must catch."""
    empty_count = n_cons if empty_count is None else empty_count
    q_full = MBar(1)
    kv_full = [MBar(1) for _ in range(stages)]
    kv_empty = [MBar(empty_count) for _ in range(stages)]
    slot = [None] * stages          # which tile's bytes the slot holds
    inflight = []                   # issued TMA loads that have not landed: ("Q", None) / (j, s)
    flags, released, log = set(), set(), []
    seg_of = []
    if segs is not None:
        for g, n in enumerate(segs):
            seg_of += [g] * n
        assert len(seg_of) == n_kv

    def producer():
        if n_kv == 0:
            return
        inflight.append(("Q", None))
        ready = -1
        for j in range(n_kv):
            s, ph = j % stages, (j // stages) & 1
            if segs is not None and seg_of[j] != ready:
                g = seg_of[j]
                yield lambda g=g: g in flags
                log.append(("flag_seen", g))
                ready = seg_of[j]
            yield lambda s=s, ph=ph: kv_empty[s].passed(ph if producer_parity_bug else ph ^ 1)
            if j >= stages:
                for w in range(n_cons):
                    if (w, j - stages) not in released:
                        raise Aliasing(f"tile {j} issued into slot {s} before warpgroup {w} released tile {j - stages}")
            log.append(("load", j))
            inflight.append((j, s))
            yield None

    def tma():
        while True:
            if not inflight:
                yield lambda: bool(inflight)      # idle until a load is issued
                continue
            j, s = inflight.pop(rng.randrange(len(inflight)))
            if j == "Q":
                log.append(("Q_landed", 0))
                q_full.arrive()
            else:
                slot[s] = j
                log.append(("landed", j))
                kv_full[s].arrive()
            yield None

    def copier():                   # peer copies of the segments land in any order, each followed by its flag
        order = list(range(len(segs or [])))
        rng.shuffle(order)
        for g in order:
            yield None
            flags.add(g)
            log.append(("flag", g))

    def consumer(w):
        if n_kv > 0:
            yield lambda: q_full.passed(0)
        for j in range(n_kv):
            s = j % stages
            yield lambda s=s, j=j: kv_full[s].passed((j // stages) & 1)
            if slot[s] != j:
                raise Aliasing(f"warpgroup {w} waited for tile {j} and found slot {s} holding {slot[s]}")
            log.append(("qk", w, j))
            yield None                                                  # softmax; QK / PV wgmma read the slot
            if slot[s] != j:
                raise Aliasing(f"slot {s} refilled under warpgroup {w}'s MMAs of tile {j}")
            log.append(("pv", w, j))
            released.add((w, j))
            kv_empty[s].arrive()
        log.append(("epilogue", w))

    agents = {"producer": producer(), "tma": tma(), "copier": copier()}
    agents.update({f"wg{w}": consumer(w) for w in range(n_cons)})
    background = {"tma", "copier"}
    waiting, live, steps = {}, set(agents), 0
    while live - background or inflight:
        steps += 1
        if steps > 50000:
            raise Deadlock("livelock")
        runnable = [a for a in live if a not in waiting or waiting[a]()]
        if not [a for a in runnable if a not in background] and not inflight and "copier" not in runnable:
            raise Deadlock(f"deadlock at n_kv={n_kv}: waiting {sorted(waiting)}; log tail {log[-8:]}")
        a = rng.choice(runnable)
        waiting.pop(a, None)
        try:
            r = next(agents[a])
        except StopIteration:
            live.discard(a)
            continue
        if callable(r):
            waiting[a] = r
    return log


def check(n_kv, log, stages=6, n_cons=2, segs=None):
    pos = {e: i for i, e in enumerate(log)}
    for j in range(n_kv):
        for w in range(n_cons):
            assert pos[("landed", j)] < pos[("qk", w, j)] < pos[("pv", w, j)] < pos[("epilogue", w)]
            if j + stages < n_kv:
                assert pos[("pv", w, j)] < pos[("load", j + stages)]
        assert pos[("load", j)] < pos[("landed", j)]
    if segs is not None:
        g0 = 0
        for g, n in enumerate(segs):
            assert pos[("flag", g)] < pos[("flag_seen", g)] < pos[("load", g0)]
            g0 += n
    if n_kv == 0:
        assert not [e for e in log if e[0] in ("load", "qk")]


def run_many(n_kv, trials, seed, **kw):
    rng = random.Random(seed)
    for _ in range(trials):
        check(n_kv, simulate(n_kv, rng, **kw), kw.get("stages", 6), kw.get("n_cons", 2), kw.get("segs"))


class Starving(random.Random):
    """Scheduler that picks `starved` only when it is the only runnable agent."""

    def __init__(self, seed, starved):
        super().__init__(seed)
        self.starved = starved

    def choice(self, seq):
        rest = [a for a in seq if a != self.starved] if seq and isinstance(seq[0], str) else seq
        return super().choice(rest if rest else seq)


@pytest.mark.parametrize("stages", [1, 2, 3, 6])
@pytest.mark.parametrize("n_kv", list(range(0, 14)))
def test_ring_no_deadlock_and_ordering(n_kv, stages):
    """Every ring depth up to the kernel's (6): each slot is reused many times, so the parity waits are exercised across phases."""
    run_many(n_kv, 60, 1234 + 7 * n_kv + stages, stages=stages)


@pytest.mark.parametrize("segs", [[2], [2, 2], [2, 2, 2, 2], [4, 4, 4], [8, 8], [1, 1, 1, 1, 1]])
def test_segment_flags_gate_the_loads(segs):
    """Fused sequence-parallel gather: the producer polls the flag of the segment of the tile it is about to load (once per
    segment, `ready_seg`); the copy engine raises the flags in any order."""
    for stages in (2, 6):
        run_many(sum(segs), 60, 99 + sum(segs) + stages, stages=stages, segs=segs)


def test_starved_agents_do_not_alias():
    """One role at a time runs only when nothing else can: the other warpgroup may run ahead by at most the ring depth and never
    finds a refilled slot; a starved producer, TMA engine or copy engine only delays."""
    for starved in ["producer", "wg0", "wg1", "tma", "copier"]:
        for n_kv, segs in ((1, None), (5, None), (13, None), (8, [2, 2, 2, 2])):
            for stages in (2, 6):
                for seed in range(8):
                    check(n_kv, simulate(n_kv, Starving(seed, starved), stages=stages, segs=segs), stages=stages, segs=segs)


def test_protocol_errors_are_caught():
    """The model has to see the errors it rules out: kv_empty released by ONE warpgroup instead of both (the producer refills a
    slot the other warpgroup still reads, or a waiter is overtaken by two phases and blocks), and the producer waiting for
    kv_empty on the wrong parity (it blocks on the first pass through the ring)."""
    rng = random.Random(7)
    caught = deadlock = 0
    for n_kv in (3, 5, 8):
        for _ in range(200):
            try:
                check(n_kv, simulate(n_kv, rng, stages=2, empty_count=1), stages=2)
            except (Aliasing, Deadlock):
                caught += 1
        try:
            simulate(n_kv, rng, stages=2, producer_parity_bug=True)
        except Deadlock:
            deadlock += 1
    assert caught > 0 and deadlock == 3
