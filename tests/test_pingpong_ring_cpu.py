"""CPU replay of the ping-pong schedule's barrier bookkeeping in conv_gemm_kernel (csrc/conv_gemm.cu).

The actors of one CTA are stepped in random interleavings, with TMA fills landing in random order:
the operand producer (its loop, including the weight prefetch before the dependency wait and the
rewind over those stages), the two consumer warpgroups (tile j belongs to warpgroup j & 1; the
k-loops take turns through the two named barriers) and the auxiliary producer of the residual
instance (two landing slots per warpgroup).  mbarriers are modelled with their phase parity, so a
wait on the wrong parity passes early or never.  Every consumer wait must see exactly the fill it
expects, every stage fill must be released once by the warpgroup that read it, and no
interleaving may deadlock."""
import random

import pytest


class MBar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, 0, 0   # phase: completed phases
        self.content = None   # what the last completed phase delivered

    def ready(self, parity):   # mbarrier.try_wait.parity
        return (self.phase & 1) != parity

    def arrive(self, content=None):
        self.pending += 1
        if self.pending == self.count:
            self.pending, self.phase, self.content = 0, self.phase + 1, content


def producer(S, k_iters, n_tiles, full, empty, landed):
    """Operand producer, line by line as in the kernel (kEarlyW: inference instances)."""
    n_pre = min(k_iters, S)
    mode = 0 if n_pre > 0 else 2
    stage = phase = it = 0
    j = 0
    fill = 0   # index of the next fill (mode 1 adds the A halves to fills 0 .. n_pre - 1)
    while True:
        if mode != 1:   # wait for the slot, expect the stage's bytes, load W
            yield lambda s=stage, ph=phase: empty[s].ready(ph ^ 1)
            assert stage not in landed
            landed[stage] = {"g": fill, "issued": 1, "got": 0}
            fill += 1
        if mode != 0:   # load A
            landed[stage]["issued"] += 1
        stage += 1
        if stage == S:
            stage, phase = 0, phase ^ 1
        it += 1
        if mode == 0 and it == n_pre:
            mode, it, stage, phase = 1, 0, 0, 0
        elif mode == 1 and it == n_pre:
            mode = 2
        if it == k_iters:
            j += 1
            if j >= n_tiles:
                return
            it = 0


def aux_producer(bpt, n_tiles, rfull, rempty, rlanded):
    filled = [0, 0]
    for j in range(n_tiles):
        g = j & 1
        for sb in range(bpt):
            n = filled[g]
            slot = 2 * g + (n & 1)
            yield lambda s=slot, ph=((n >> 1) & 1) ^ 1: rempty[s].ready(ph)
            rlanded[slot] = (j, sb)
            filled[g] += 1


def consumer(wg, S, k_iters, n_tiles, bpt, res, full, empty, rfull, rempty, order, log):
    res_seen = 0
    for j in range(wg, n_tiles, 2):
        fill = j * k_iters
        stage, phase = fill % S, (fill // S) & 1
        if j > 0:
            yield lambda: order[wg] > 0           # bar.sync 8 + wg
            order[wg] -= 1
        prev = None
        for it in range(k_iters):
            yield lambda s=stage, ph=phase: full[s].ready(ph)
            assert full[stage].content == fill + it, (wg, j, it, full[stage].content)
            log["read"].append(fill + it)
            if it > 0:
                empty[prev].arrive()
                log["released"].append((wg, prev_g))
            prev, prev_g = stage, fill + it
            stage += 1
            if stage == S:
                stage, phase = 0, phase ^ 1
        if j + 1 < n_tiles:
            assert order[1 - wg] == 0, "an order barrier arrival would merge two generations"
            order[1 - wg] += 1                     # bar.arrive 9 - wg
        empty[prev].arrive()
        log["released"].append((wg, prev_g))
        if res:
            for sb in range(bpt):
                slot = 2 * wg + (res_seen & 1)
                yield lambda s=slot, ph=(res_seen >> 1) & 1: rfull[s].ready(ph)
                assert rfull[slot].content == (j, sb), (wg, j, sb, rfull[slot].content)
                res_seen += 1
            for sb in range(bpt):
                rempty[2 * wg + ((res_seen - bpt + sb) & 1)].arrive()
        log["tiles"].append((wg, j))


def replay(S, k_iters, n_tiles, bpt, res, seed):
    rng = random.Random(seed)
    full = [MBar(1) for _ in range(S)]
    empty = [MBar(1) for _ in range(S)]   # the 4 warps of the reading warpgroup, as one arrival
    rfull = [MBar(1) for _ in range(4)]
    rempty = [MBar(1) for _ in range(4)]
    landed, rlanded, order = {}, {}, [0, 0]
    log = {"read": [], "released": [], "tiles": []}
    actors = [producer(S, k_iters, n_tiles, full, empty, landed)]
    actors += [consumer(g, S, k_iters, n_tiles, bpt, res, full, empty, rfull, rempty, order, log)
               for g in (0, 1)]
    if res:
        actors.append(aux_producer(bpt, n_tiles, rfull, rempty, rlanded))
    waits = {}
    for a in actors:
        try:
            waits[a] = next(a)
        except StopIteration:
            pass
    while waits or landed or rlanded:
        choices = [("actor", a) for a, w in waits.items() if w()]
        choices += [("land", s) for s, t in landed.items() if t["got"] < t["issued"]]
        choices += [("rland", s) for s in rlanded]
        assert choices, "deadlock"
        kind, x = rng.choice(choices)
        if kind == "land":   # one half (W or A) of a stage lands; the fill completes with both
            t = landed[x]
            t["got"] += 1
            if t["got"] == 2:
                del landed[x]
                full[x].arrive(t["g"])
            continue
        if kind == "rland":
            rfull[x].arrive(rlanded.pop(x))
            continue
        try:
            waits[x] = x.send(None)
        except StopIteration:
            del waits[x]
    total = n_tiles * k_iters
    assert sorted(log["read"]) == list(range(total))
    released = sorted(g for _, g in log["released"])
    assert released == list(range(total)), "every stage fill is released exactly once"
    for wg, g in log["released"]:
        assert (g // k_iters) & 1 == wg, "a fill is released by the warpgroup that read it"
    assert sorted(j for _, j in log["tiles"]) == list(range(n_tiles))


@pytest.mark.parametrize("k_iters", [1, 2, 16, 48])
@pytest.mark.parametrize("stages", [4, 5, 6])
@pytest.mark.parametrize("res,bpt", [(False, 2), (True, 1), (True, 2)])
def test_pingpong_ring_replay(k_iters, stages, res, bpt):
    # tiles per CTA: 1 (the schedule is only chosen from 2 on, but must still be sound), 2, 3, and
    # the larger odd / even counts of the flagship's early layers
    for n_tiles in (1, 2, 3, 5, 14):
        for seed in range(6 if k_iters < 48 else 2):
            replay(stages, k_iters, n_tiles, bpt, res, seed)


def tiles_per_cta(total, sms):
    grid = min(total, sms)
    return [len(range(b, total, grid)) for b in range(grid)]


def test_tile_lists_of_grids():
    # the CTA tile counts the replay covers arise from real grids: odd totals, 1 to 3 per CTA
    assert set(tiles_per_cta(100, 132)) == {1}
    assert set(tiles_per_cta(264, 132)) == {2}
    assert set(tiles_per_cta(392, 132)) == {2, 3}
    assert set(tiles_per_cta(235, 132)) == {1, 2}
    assert set(tiles_per_cta(1728, 132)) == {13, 14}
