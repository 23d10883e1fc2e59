"""CPU model of the two-pass schedule of the forward solve of `mlpg_fwd_as_kernel` (csrc/nnk_mlpg_as.cuh).

Pass 1 is the forward sweep: NA assemblers publish band-row tiles 0 .. npb-1 through a PB ring of ND slots.
A CTA barrier ends it.  Pass 2 is the segment replay: AS_NA_B of the assemblers publish the replay sequence (the
segments from the last to the first, tiles ascending inside each, padded to an even count by a ghost tile)
through a second PB ring of AS_ND_B slots with its own barriers.  Each assembler's input-stage ring (NSA stages,
refilled NSA tiles ahead, a tile without rows completing its stage with a plain arrive) runs on across both
passes.  Every wait sees only the parity of a phase, like an mbarrier."""
import random

from test_ring_protocol_model_cpu import Bar

NA, ND, NA_B, ND_B = 3, 6, 2, 3


def replay_sequence(npb, KT, pairs=True):
    """Tile k of every position n of the replay sequence (`bw_tile`; npb itself is the ghost tile)."""
    nseg = (npb + KT - 1) // KT
    nbk = (npb + 1) & ~1 if pairs else npb
    nlast = nbk - (nseg - 1) * KT
    return [(nseg - 1) * KT + n if n < nlast else (nseg - 2 - (n - nlast) // KT) * KT + (n - nlast) % KT
            for n in range(nbk)]


def _owned(role, na, n_tiles):
    out, n = [], 2 * role
    while n < n_tiles:
        out.append(n)
        n = n + 1 if n % 2 == 0 else n - 1 + 2 * na
    return out


def simulate(npb, KT, NSA, seed, bias, nd_b=ND_B, na_b=NA_B):
    """One random interleaving of both passes (one chain group).  "ok", "corrupt" or "deadlock"."""
    rng = random.Random(seed)
    seq = replay_sequence(npb, KT)
    passes = [(NA, ND, list(range(npb))), (na_b, nd_b, seq)]
    stage_full = [[Bar() for _ in range(NSA)] for _ in range(NA)]
    stage_tile = [[None] * NSA for _ in range(NA)]
    st = [0] * NA                       # running stage index of each assembler (both passes)
    pending = [dict() for _ in range(NA)]  # stage -> tile whose copy is in flight
    used = [[0] * NSA for _ in range(NA)]  # completed uses of each stage: the parity its next wait expects
    for na, nd, tiles in passes:
        full = [Bar() for _ in range(nd)]
        empty = [Bar() for _ in range(nd)]
        slot, unread = [None] * nd, [False] * nd
        queues = [_owned(r, na, len(tiles)) if r < na else [] for r in range(NA)]
        pos = [0] * NA
        for r in range(na):             # prologue: the first NSA tiles of the pass
            for i, n in enumerate(queues[r][:NSA]):
                pending[r][(st[r] + i) % NSA] = n
        nxt = 0
        while nxt < len(tiles):
            run = []
            for r in range(na):
                for s, n in list(pending[r].items()):  # copies land at any time
                    if rng.random() < 0.5:
                        stage_tile[r][s] = n
                        stage_full[r][s].arrive()
                        del pending[r][s]
                if pos[r] < len(queues[r]):
                    n = queues[r][pos[r]]
                    s = st[r]
                    if empty[n % nd].passes(((n // nd) & 1) ^ 1) and stage_full[r][s].passes(used[r][s] & 1):
                        run.append(("p", r))
            if full[nxt % nd].passes((nxt // nd) & 1):
                run.append(("c", 0))
            if not run:
                if any(pending[r] for r in range(na)):
                    continue
                return "deadlock"
            kind, r = rng.choices(run, [bias if a[0] == "p" else 1.0 for a in run])[0]
            if kind == "p":
                n = queues[r][pos[r]]
                s = st[r]
                if stage_tile[r][s] != n:
                    return "corrupt"    # converted the wrong rows
                used[r][s] += 1
                if pos[r] + NSA < len(queues[r]):
                    pending[r][s] = queues[r][pos[r] + NSA]
                if unread[n % nd]:
                    return "corrupt"    # an undrained band-row tile is overwritten
                slot[n % nd], unread[n % nd] = n, True
                full[n % nd].arrive()
                pos[r] += 1
                st[r] = (s + 1) % NSA
            else:
                if slot[nxt % nd] != nxt:
                    return "corrupt"
                unread[nxt % nd] = False
                empty[nxt % nd].arrive()
                nxt += 1
        # the pass boundary is a CTA barrier: every warp has finished the pass here
    return "ok"


def outcomes(npb, KT=8, NSA=2, runs=40, biases=(0.05, 1.0, 16.0), **kw):
    seen = set()
    for seed in range(runs):
        for b in biases:
            seen.add(simulate(npb, KT, NSA, seed, b, **kw))
    return seen


def test_replay_sequence_covers_every_tile_once_in_whole_pairs():
    for KT in (4, 8):
        for npb in range(1, 90):
            seq = replay_sequence(npb, KT)
            real = [k for k in seq if k < npb]
            assert sorted(real) == list(range(npb)) and len(seq) - len(real) == npb % 2
            for m in range(0, len(seq), 2):  # a pair is two consecutive tiles of one segment
                assert seq[m] % 2 == 0 and seq[m + 1] == seq[m] + 1 and seq[m] // KT == seq[m + 1] // KT
            segs = [k // KT for k in seq]
            assert segs == sorted(segs, reverse=True)  # segments from the last to the first


def test_two_pass_schedule_is_safe():
    for npb in (1, 2, 3, 7, 8, 9, 16, 17, 40, 41):
        for NSA in (1, 2):
            assert outcomes(npb, NSA=NSA) == {"ok"}, (npb, NSA)


def test_replay_ring_shallower_than_the_producer_stride_is_unsafe():
    # three replay assemblers on a 3-slot ring: stride 2 * 3 - 1 = 5 > 3
    assert outcomes(41, NSA=1, na_b=3, nd_b=3) & {"corrupt", "deadlock"}
