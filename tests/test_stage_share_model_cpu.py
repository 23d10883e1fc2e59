"""CPU model of the shared input stages of the G = 2 `mlpg_fwd_as_kernel` (csrc/nnk_mlpg_as.cuh): the two
assembler warps of a pair (one per chain group) read every tile of one ring of NSA stages.  Each warp waits
on the stage's `in_full` barrier with a parity-only wait, reads the rows, then releases the stage by bumping
a per-stage counter; the release that finds an odd count (the second one of that use) issues the bulk copy
of the tile NSA turns later into the same stage.  The copy lands at some later time and completes the
barrier's phase.  Under random interleavings the model checks that no copy overwrites a stage a reader has
not released, that every use is refilled exactly once, and that every reader reads the tile it expects."""
import random


class Bar(object):
    """An mbarrier reduced to its phase counter: wait(parity) passes iff the phase of that parity is complete."""

    def __init__(self):
        self.done = 0

    def passes(self, parity):
        return (self.done & 1) != parity

    def arrive(self):
        self.done += 1


def simulate(NSA, n_tiles, readers, seed, policy="last"):
    """One random interleaving of `readers` warps over `n_tiles` tiles of one pair.  `policy`: "last" (the
    kernel: the second release issues), "first" (the first release issues) or "each" (every release issues).
    Returns "ok", "early" (a stage overwritten before every reader released it), "wrong" (a reader saw
    another tile), "double" (a use refilled twice) or "deadlock" (a refill never issued)."""
    rng = random.Random(seed)
    full = [Bar() for _ in range(NSA)]
    cnt = [0] * NSA
    content = [None] * NSA
    holders = [set() for _ in range(NSA)]  # readers that have not yet released the stage's current tile
    pending = []  # bulk copies in flight: (stage, tile)
    issued = {}   # tile -> number of copies issued
    pos = [0] * readers
    par = [0] * readers

    def issue(tile):
        if tile >= n_tiles:
            return
        issued[tile] = issued.get(tile, 0) + 1
        pending.append((tile % NSA, tile))

    for t in range(min(NSA, n_tiles)):  # the prologue: half 0, lane 0
        issue(t)
    while min(pos) < n_tiles:
        acts = [("dma", i) for i in range(len(pending))]
        for r in range(readers):
            if pos[r] < n_tiles and full[pos[r] % NSA].passes(par[r]):
                acts.append(("read", r))
        if not acts:
            return "deadlock"
        kind, i = rng.choice(acts)
        if kind == "dma":
            s, tile = pending.pop(i)
            if holders[s]:
                return "early"
            content[s] = tile
            holders[s] = set(range(readers))
            full[s].arrive()
            continue
        r = i
        k = pos[r]
        s = k % NSA
        if content[s] != k or r not in holders[s]:
            return "wrong"
        holders[s].discard(r)  # the rows are in registers: release
        prior = cnt[s]
        cnt[s] += 1
        last = readers == 1 or (prior & 1) == 1
        if policy == "each" or (policy == "last" and last) or (policy == "first" and not last):
            issue(k + NSA)
        pos[r] += 1
        if s == NSA - 1:
            par[r] ^= 1
    if any(n != 1 for n in issued.values()) or len(issued) != n_tiles:
        return "double"
    return "ok"


def outcomes(NSA, readers, policy="last", runs=300, n_tiles=40):
    return {simulate(NSA, n_tiles, readers, seed, policy) for seed in range(runs)}


def test_last_release_issues_every_refill_exactly_once():
    for NSA in (1, 2, 3):
        assert outcomes(NSA, readers=2) == {"ok"}, NSA
        assert outcomes(NSA, readers=1) == {"ok"}, NSA  # the absent second group of an odd group count


def test_first_release_issuing_overwrites_a_stage_in_use():
    assert "early" in outcomes(2, readers=2, policy="first")


def test_every_release_issuing_refills_twice():
    assert outcomes(2, readers=2, policy="each") - {"ok"}
