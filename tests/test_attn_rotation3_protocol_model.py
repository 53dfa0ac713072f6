"""Model check (CPU) of the three-way turn rotation of the forward kernel's three-consumer form (csrc/attn.cu, kNC = 3: the dense
INT8+FP8 kernel at head dim 128, 192-row Q tiles).  One TMA producer over the kStages-deep K/V^T ring and three consumer
warpgroups, each with n_kv + 1 tensor-core phases (QK(0); PV(j-1) + QK(j) for j = 1..n_kv-1; PV(n_kv-1)), issued in turn.

Named barrier 1 + w is warpgroup w's turn: w waits on it with bar.sync before a phase, and its predecessor (w + 2) % 3 arrives
on it with bar.arrive once its phase is issued; each completion takes one sync and one arrival (2 x 128 threads).  Warpgroup 2
arrives on warpgroup 0's barrier once before its loop, so warpgroup 0 goes first; warpgroups 0 and 1 hand over after every phase,
warpgroup 2 after every phase but its last.  Every warpgroup runs all n_kv + 1 phases, also when its 64 rows all lie past the end
of the sequence (the last Q tile of a sequence whose length is not a multiple of 192).  Slot j-1 is released after the wait of
the phase that issued PV(j-1).  Random interleavings, with the TMA engine landing loads in any order.  Checked, for n_kv = 0..9:
  * no deadlock (every agent terminates),
  * the GEMM phases go round 0, 1, 2, 0, 1, 2, ...,
  * no named-barrier arrival is unmatched: no warpgroup arrives twice in one barrier phase, and none is pending at exit,
  * a slot is refilled only after all three warpgroups released it, and holds the tile a phase reads until its MMAs end.
The model also has to catch the wrong variants: no first hand-over (deadlock), a hand-over after warpgroup 2's last phase (an
arrival left over at exit), and a warpgroup past the end of the sequence that skips its phases (deadlock)."""
import random

import pytest

from test_attn_pingpong_protocol_model import NamedBar, Unmatched
from test_attn_ring_protocol_model import MBar, Aliasing, Deadlock, Starving

NC = 3


def simulate(n_kv, rng, stages=6, valid_wgs=NC, first_turn=True, last_arrive=False, skip_past_end=False):
    """Runs one random schedule; returns (log, order of GEMM phases by warpgroup, the turn barriers).
    valid_wgs: warpgroups whose rows start inside the sequence (a partial last Q tile has fewer than three).
    first_turn=False / last_arrive=True / skip_past_end=True: deliberately wrong protocols the checks must catch."""
    q_full = MBar(1)
    kv_full = [MBar(1) for _ in range(stages)]
    kv_empty = [MBar(NC) for _ in range(stages)]
    turn = [NamedBar(1 + w) for w in range(NC)]      # turn[w]: named barrier 1 + w
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
                for w in range(NC):
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
        if n_kv == 0 or (skip_past_end and w >= valid_wgs):
            return
        yield lambda: q_full.passed(0)
        if w == NC - 1 and first_turn:
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
            yield None                                            # PV half 0 lands and is folded: the turn is still held
            if w != NC - 1 or ph < n_kv or last_arrive:
                turn[(w + 1) % NC].arrive(w)
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

    agents = {"producer": producer(), "tma": tma(), **{f"wg{w}": consumer(w) for w in range(NC)}}
    waiting, live, steps = {}, set(agents), 0
    while live - {"tma"} or inflight:
        steps += 1
        if steps > 80000:
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
    assert order == list(range(NC)) * phases, f"GEMM phases out of turn: {order}"
    for bar in turn:
        if bar.arrived:
            raise Unmatched(f"arrival of warpgroup {bar.arrived} left over at exit on barrier {bar.name}")
        assert bar.gen == phases
    pos = {e: i for i, e in enumerate(log)}
    for j in range(n_kv):
        for w in range(NC):
            assert pos[("landed", j)] < pos[("phase", w, j)] < pos[("release", w, j)] < pos[("epilogue", w)]
            if j + stages < n_kv:
                assert pos[("release", w, j)] < pos[("load", j + stages)]
    if n_kv == 0:
        assert not log


@pytest.mark.parametrize("stages", [2, 6])
@pytest.mark.parametrize("n_kv", list(range(0, 10)))
def test_rotation_goes_round_without_deadlock(n_kv, stages):
    rng = random.Random(8765 + 13 * n_kv + stages)
    for _ in range(150):
        check(n_kv, simulate(n_kv, rng, stages=stages), stages)


@pytest.mark.parametrize("valid_wgs", [1, 2])
@pytest.mark.parametrize("n_kv", [0, 1, 2, 5])
def test_partial_last_tile(n_kv, valid_wgs):
    """A last Q tile with only 64 or 128 rows inside the sequence: the warpgroups past the end still take and pass their turns."""
    rng = random.Random(99 + n_kv + valid_wgs)
    for _ in range(100):
        check(n_kv, simulate(n_kv, rng, valid_wgs=valid_wgs))


def test_starved_agents():
    """One role at a time runs only when nothing else can: the rotation still goes round and never aliases a slot."""
    for starved in ["producer", "tma", "wg0", "wg1", "wg2"]:
        for n_kv in (1, 2, 7, 9):
            for seed in range(8):
                check(n_kv, simulate(n_kv, Starving(seed, starved)))


def test_wrong_hand_over_is_caught():
    rng = random.Random(23)
    for n_kv in (1, 2, 4, 9):
        with pytest.raises(Deadlock):
            simulate(n_kv, rng, first_turn=False)
        with pytest.raises(Unmatched):
            check(n_kv, simulate(n_kv, rng, last_arrive=True))
        with pytest.raises(Deadlock):
            simulate(n_kv, rng, valid_wgs=2, skip_past_end=True)
