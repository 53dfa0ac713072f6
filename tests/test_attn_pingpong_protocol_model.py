"""Model check (CPU) of the ping-pong schedule of the forward kernel's consumer loop (csrc/attn.cu): one TMA producer over the
kStages-deep K/V^T ring, and two consumer warpgroups whose loop is rotated so that each has n_kv + 1 tensor-core phases
(QK(0); PV(j-1) + QK(j) for j = 1..n_kv-1; PV(n_kv-1)) and takes turns at issuing them through two named barriers.

Named barrier 1 + w is warpgroup w's turn: w waits on it with bar.sync before a phase, the other warpgroup arrives on it with
bar.arrive right after its commit; each completion takes one sync and one arrival (2 x 128 threads).  Warpgroup 1 arrives once
before its loop so warpgroup 0 goes first; warpgroup 0 arrives after every phase, warpgroup 1 after every phase but its last.
A warpgroup waits on kv_full(j) before it takes the turn, and releases slot j-1 (kv_empty) after the wait of the phase that
issued PV(j-1).  Random interleavings, with the TMA engine landing loads in any order.  Checked, for n_kv = 0..9:
  * no deadlock (every agent terminates),
  * the GEMM phases strictly alternate 0, 1, 0, 1, ...,
  * no named-barrier arrival is unmatched: no warpgroup arrives twice in one barrier phase, and none is pending at exit,
  * a slot is refilled only after both warpgroups released it, and holds the tile a phase reads until that phase's MMAs end.
The model also has to catch the wrong variants: no first hand-over (deadlock), and a hand-over after warpgroup 1's last phase
(an arrival left over at exit)."""
import random

import pytest

from test_attn_ring_protocol_model import MBar, Aliasing, Deadlock, Starving


class Unmatched(AssertionError):
    pass


class NamedBar:
    """bar.sync / bar.arrive with an expected count of two warpgroups (256 threads)."""

    def __init__(self, name, count=2):
        self.name, self.count, self.arrived, self.gen = name, count, [], 0

    def arrive(self, who):
        if who in self.arrived:
            raise Unmatched(f"warpgroup {who} arrived twice in one phase of barrier {self.name}")
        self.arrived.append(who)
        if len(self.arrived) == self.count:
            self.arrived, self.gen = [], self.gen + 1

    def sync(self, who):   # generator: arrive, then wait for the phase to complete
        g = self.gen
        self.arrive(who)
        yield lambda: self.gen != g


def simulate(n_kv, rng, stages=6, first_turn=True, last_arrive=False):
    """Runs one random schedule; returns (log, order of GEMM phases by warpgroup, the two turn barriers).
    first_turn=False / last_arrive=True: deliberately wrong hand-over counts the checks must catch."""
    q_full = MBar(1)
    kv_full = [MBar(1) for _ in range(stages)]
    kv_empty = [MBar(2) for _ in range(stages)]
    turn = [NamedBar(1), NamedBar(2)]        # turn[w]: named barrier 1 + w
    slot = [None] * stages
    inflight, released, log, order = [], set(), [], []

    def producer():
        if n_kv == 0:
            return
        inflight.append(("Q", None))
        for j in range(n_kv):
            s, ph = j % stages, (j // stages) & 1
            yield lambda s=s, ph=ph: kv_empty[s].passed(ph ^ 1)
            if j >= stages:
                for w in range(2):
                    if (w, j - stages) not in released:
                        raise Aliasing(f"tile {j} issued into slot {s} before warpgroup {w} released tile {j - stages}")
            log.append(("load", j))
            inflight.append((j, s))
            yield None

    def tma():
        while True:
            if not inflight:
                yield lambda: bool(inflight)
                continue
            j, s = inflight.pop(rng.randrange(len(inflight)))
            if j == "Q":
                q_full.arrive()
            else:
                slot[s] = j
                log.append(("landed", j))
                kv_full[s].arrive()
            yield None

    def consumer(w):
        if n_kv == 0:
            return
        yield lambda: q_full.passed(0)
        if w == 1 and first_turn:
            turn[0].arrive(w)
        for ph in range(n_kv + 1):
            reads = [t for t in (ph - 1, ph) if 0 <= t < n_kv]    # PV(ph-1), QK(ph)
            if ph < n_kv:
                yield lambda j=ph: kv_full[j % stages].passed((j // stages) & 1)
            yield from turn[w].sync(w)
            order.append(w)
            log.append(("phase", w, ph))
            for t in reads:
                if slot[t % stages] != t:
                    raise Aliasing(f"warpgroup {w} phase {ph} found slot {t % stages} holding {slot[t % stages]}, not tile {t}")
            if w == 0 or ph < n_kv or last_arrive:
                turn[1 - w].arrive(w)
            yield None                                            # MMAs in flight: everyone else runs
            for t in reads:
                if slot[t % stages] != t:
                    raise Aliasing(f"slot {t % stages} refilled under warpgroup {w}'s MMAs of tile {t}")
            if ph > 0:
                released.add((w, ph - 1))
                log.append(("release", w, ph - 1))
                kv_empty[(ph - 1) % stages].arrive()
            yield None                                            # softmax(ph)
        log.append(("epilogue", w))

    agents = {"producer": producer(), "tma": tma(), "wg0": consumer(0), "wg1": consumer(1)}
    waiting, live, steps = {}, set(agents), 0
    while live - {"tma"} or inflight:
        steps += 1
        if steps > 50000:
            raise Deadlock("livelock")
        runnable = [a for a in live if a not in waiting or waiting[a]()]
        if not [a for a in runnable if a != "tma"] and not inflight:
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
    return log, order, turn


def check(n_kv, result, stages=6):
    log, order, turn = result
    phases = n_kv + 1 if n_kv > 0 else 0
    assert order == [0, 1] * phases, f"GEMM phases out of turn: {order}"
    for bar in turn:
        if bar.arrived:
            raise Unmatched(f"arrival of warpgroup {bar.arrived} left over at exit on barrier {bar.name}")
        assert bar.gen == phases
    pos = {e: i for i, e in enumerate(log)}
    for j in range(n_kv):
        for w in range(2):
            assert pos[("landed", j)] < pos[("phase", w, j)] < pos[("release", w, j)] < pos[("epilogue", w)]
            if j + stages < n_kv:
                assert pos[("release", w, j)] < pos[("load", j + stages)]
    if n_kv == 0:
        assert not log


@pytest.mark.parametrize("stages", [2, 6])
@pytest.mark.parametrize("n_kv", list(range(0, 10)))
def test_pingpong_alternates_without_deadlock(n_kv, stages):
    rng = random.Random(4321 + 11 * n_kv + stages)
    for _ in range(200):
        check(n_kv, simulate(n_kv, rng, stages=stages), stages)


def test_starved_agents():
    """One role at a time runs only when nothing else can: the schedule still alternates and never aliases a slot."""
    for starved in ["producer", "tma", "wg0", "wg1"]:
        for n_kv in (1, 2, 7, 9):
            for seed in range(10):
                check(n_kv, simulate(n_kv, Starving(seed, starved)))


def test_wrong_hand_over_is_caught():
    rng = random.Random(17)
    for n_kv in (1, 4, 9):
        with pytest.raises(Deadlock):
            simulate(n_kv, rng, first_turn=False)
        with pytest.raises(Unmatched):
            check(n_kv, simulate(n_kv, rng, last_arrive=True))
