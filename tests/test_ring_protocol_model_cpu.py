"""CPU model of the band-row (PB) ring protocol of csrc/nnk_mlpg_as.cuh: NA producer warps publish tiles into
ND slots, one consumer drains them in order, and -- like an mbarrier -- a wait only sees the PARITY of a
barrier's phase.  The model reproduces the root cause of the round-1 "deadlock under pytest only"
(tools/experiments/README.md): a producer whose next tile lies more than ND tiles beyond the one it was
last admitted for can pass its `pb_empty` wait on a phase that is two wraps old and overwrite an undrained
slot.  Safe iff the producers' tile stride <= ND -- the `static_assert` the kernel now carries."""
import random


class Bar(object):
    """An mbarrier reduced to its phase counter: wait(parity) passes iff the phase of that parity is complete."""

    def __init__(self):
        self.done = 0  # completed phases

    def passes(self, parity):
        return (self.done & 1) != parity  # try_wait.parity: true once the current phase's parity differs

    def arrive(self):
        self.done += 1


def _tiles_of(role, NA, n_tiles, pairs):
    if not pairs:
        return list(range(role, n_tiles, NA))
    out, k = [], 2 * role
    while k < n_tiles:
        out.append(k)
        k = k + 1 if k % 2 == 0 else k - 1 + 2 * NA
    return out


def simulate(NA, ND, n_tiles, pairs, seed, producer_bias):
    """One random interleaving.  Returns "ok", "corrupt" (a slot overwritten before it was read, or read with the
    wrong tile in it) or "deadlock"."""
    rng = random.Random(seed)
    full = [Bar() for _ in range(ND)]
    empty = [Bar() for _ in range(ND)]
    slot = [None] * ND       # tile currently stored in the slot
    unread = [False] * ND
    queues = [_tiles_of(r, NA, n_tiles, pairs) for r in range(NA)]
    pos = [0] * NA
    next_read = 0
    turn = -1
    while next_read < n_tiles:
        runnable = []
        for r in range(NA):
            if pos[r] < len(queues[r]):
                k = queues[r][pos[r]]
                if empty[k % ND].passes(((k // ND) & 1) ^ 1):  # nnk_mlpg_as.cuh: mbar_wait_parked(pb_empty + ps, ...)
                    runnable.append(("p", r))
        ps = next_read % ND
        if full[ps].passes((next_read // ND) & 1):              # solver: mbar_wait(pb_full + ps, ppar)
            runnable.append(("c", 0))
        if not runnable:
            return "deadlock"
        if producer_bias is None:  # fair round robin: every warp advances at the same pace
            turn += 1
            order = [("p", q) for q in range(NA)] + [("c", 0)]
            pick = [a for a in order[turn % len(order):] + order[:turn % len(order)] if a in runnable][0]
            kind, r = pick
        else:
            weights = [producer_bias if kind == "p" else 1.0 for kind, _ in runnable]
            kind, r = rng.choices(runnable, weights)[0]
        if kind == "p":
            k = queues[r][pos[r]]
            s = k % ND
            if unread[s]:
                return "corrupt"          # an undrained band-row tile is overwritten
            slot[s], unread[s] = k, True
            full[s].arrive()
            pos[r] += 1
        else:
            if slot[ps] != next_read:
                return "corrupt"          # the solver eliminates with the wrong rows
            unread[ps] = False
            empty[ps].arrive()
            next_read += 1
    return "ok"


def outcomes(NA, ND, pairs, runs=200, biases=(0.02, 1.0, 4.0, 16.0)):
    """Outcomes over random interleavings; `biases` = how much more often a ready producer is scheduled than
    the ready consumer (producers far ahead of the consumer is the dangerous regime)."""
    seen = set()
    for seed in range(runs):
        for bias in biases:
            seen.add(simulate(NA, ND, 60, pairs, seed, bias))
    return seen


def test_shipped_configuration_is_safe():
    assert outcomes(NA=3, ND=4, pairs=False) == {"ok"}      # stride 3 <= 4 (unpaired tiles)
    assert outcomes(NA=2, ND=4, pairs=False) == {"ok"}
    assert outcomes(NA=4, ND=4, pairs=False) == {"ok"}      # stride == ND is still covered


def test_paired_tiles_with_ring_depth_4_corrupt_or_hang():
    bad = outcomes(NA=3, ND=4, pairs=True)                   # stride 2*NA - 1 = 5 > 4: the round-1 attempt
    assert bad & {"corrupt", "deadlock"}, bad
    # ... and timing decides: while all warps advance at the same pace (the stand-alone runs) nothing goes
    # wrong; a producer that gets a few tiles ahead of its siblings (another clock / cache state) aliases
    assert outcomes(NA=3, ND=4, pairs=True, runs=1, biases=(None,)) == {"ok"}


def test_paired_tiles_with_ring_depth_6_are_safe():
    assert outcomes(NA=3, ND=6, pairs=True) == {"ok"}       # the shipped kernel (paired tiles, ND = 6)
    assert outcomes(NA=3, ND=5, pairs=True) == {"ok"}       # stride 5 <= 5


def test_stride_beyond_ring_depth_is_unsafe_without_pairs_too():
    assert outcomes(NA=5, ND=4, pairs=False) & {"corrupt", "deadlock"}
