"""The swapped-operand tap-GEMM's operand rings (csrc/gemm_tc_swap.cuh), replayed symbolically.

The A (slab) producer, the B (weight tile) producer and the two consumer warpgroups are restated as sequences of
mbarrier waits, TMA fills and arrivals in the kernel's order, including the consumers' deferred release (a group's
slots are released once the next group has been issued and wait_group 1 has completed it).  A scheduler runs them with
one warpgroup held back by a lag; the replay must always finish (no deadlock), and no fill may land in a slot that a
consumer still reads.  Paired and unpaired mode issue the same barrier sequence (a paired group is two wgmmas on the
same slots), so one model covers both; `items` is the number of tiles or pairs a CTA takes.
"""
import itertools

import pytest


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, 0, 0

    def arrive(self):
        self.pending += 1
        if self.pending == self.count:
            self.pending = 0
            self.phase += 1

    def passed(self, parity):  # mbarrier.try_wait.parity: the phase of this parity has completed
        return (self.phase & 1) != parity


def producer(kind, cfg):
    """A: one slab per (item, group, chunk, plane); B: one weight tile per (item, group, chunk, tap, plane)"""
    n = cfg["a_slots"] if kind == "a" else cfg["b_slots"]
    s = p = 0
    for _ in range(cfg["items"]):
        for _g in range(cfg["ngroups"]):
            for _ch in range(cfg["kchunks"]):
                for _ in range(cfg["planes"] * (1 if kind == "a" else cfg["taps"])):
                    yield ("wait", kind + "_empty", s, p ^ 1)
                    yield ("fill", kind, s)
                    s += 1
                    if s == n:
                        s, p = 0, p ^ 1


def consumer(wg, cfg):
    NA, NB = cfg["a_slots"], cfg["b_slots"]
    sa = pa = sb = pb = 0
    for _ in range(cfg["items"]):
        rel = {"a": -1, "b": -1}

        def group(reads, last_b, last_a):
            yield ("issue", wg, reads)
            # wait_group 1: the previous group has completed; its last-read slots are released
            for k in ("b", "a"):
                if rel[k] >= 0:
                    yield ("arrive", k + "_empty", rel[k], wg)
            rel["b"], rel["a"] = last_b, last_a

        for _g in range(cfg["ngroups"]):
            for _ch in range(cfg["kchunks"]):
                sa_hi, pa_hi = sa, pa
                sa += 1
                if sa == NA:
                    sa, pa = 0, pa ^ 1
                sa_lo, pa_lo = sa, pa
                if cfg["planes"] == 2:
                    sa += 1
                    if sa == NA:
                        sa, pa = 0, pa ^ 1
                yield ("wait", "a_full", sa_hi, pa_hi)
                for tp in range(cfg["taps"]):
                    last = tp == cfg["taps"] - 1
                    if cfg["planes"] == 1:
                        yield ("wait", "b_full", sb, pb)
                        yield from group([("a", sa_hi), ("b", sb)], sb, sa_hi if last else -1)
                        sb += 1
                        if sb == NB:
                            sb, pb = 0, pb ^ 1
                    else:
                        yield ("wait", "b_full", sb, pb)
                        yield from group([("a", sa_hi), ("b", sb)], sb, -1)
                        sb += 1
                        if sb == NB:
                            sb, pb = 0, pb ^ 1
                        yield ("wait", "b_full", sb, pb)
                        yield from group([("a", sa_hi), ("b", sb)], -1, sa_hi if last else -1)
                        if tp == 0:
                            yield ("wait", "a_full", sa_lo, pa_lo)
                        yield from group([("a", sa_lo), ("b", sb)], sb, sa_lo if last else -1)
                        sb += 1
                        if sb == NB:
                            sb, pb = 0, pb ^ 1
        yield ("drain", wg)  # wait_group 0, then the last group's releases
        for k in ("b", "a"):
            if rel[k] >= 0:
                yield ("arrive", k + "_empty", rel[k], wg)


def replay(cfg, lag):
    """run the four agents; warpgroup 1 may only step when it is `lag` steps behind warpgroup 0 or warpgroup 0 cannot
    step.  Returns True when every agent finished, False on deadlock."""
    bars = {}
    for k, n in (("a", cfg["a_slots"]), ("b", cfg["b_slots"])):
        bars[k + "_full"] = [Bar(1) for _ in range(n)]
        bars[k + "_empty"] = [Bar(2) for _ in range(n)]  # every consumer thread of both warpgroups
    filled = {"a": [None] * cfg["a_slots"], "b": [None] * cfg["b_slots"]}  # fill id a slot holds
    fills = {"a": 0, "b": 0}
    live = [{"a": {}, "b": {}} for _ in range(2)]  # per warpgroup: slot -> fill id it still reads
    agents = {"A": producer("a", cfg), "B": producer("b", cfg), 0: consumer(0, cfg), 1: consumer(1, cfg)}
    head = {k: next(g) for k, g in agents.items()}
    steps = {0: 0, 1: 0}

    def ready(op):
        return op[0] != "wait" or bars[op[1]][op[2]].passed(op[3])

    def do(op):
        if op[0] == "fill":
            k, s = op[1], op[2]
            for wg in (0, 1):
                assert s not in live[wg][k], f"{cfg}: fill of {k} slot {s} while warpgroup {wg} reads it"
            filled[k][s] = fills[k]
            fills[k] += 1
            bars[k + "_full"][s].arrive()
        elif op[0] == "issue":
            for k, s in op[2]:
                assert filled[k][s] is not None
                prev = live[op[1]][k].setdefault(s, filled[k][s])
                assert prev == filled[k][s], f"{cfg}: {k} slot {s} refilled under a reader"
        elif op[0] == "arrive":
            live[op[3]][op[1][0]].pop(op[2])
            bars[op[1]][op[2]].arrive()

    while head:
        order = ["A", "B", 0, 1] if steps[1] + lag <= steps[0] or 0 not in head else ["A", "B", 0]
        if not any(k in head and ready(head[k]) for k in order):
            order = ["A", "B", 0, 1]  # the held-back warpgroup steps when nothing else can
        for k in order:
            if k in head and ready(head[k]):
                do(head[k])
                if k in steps:
                    steps[k] += 1
                try:
                    head[k] = next(agents[k])
                except StopIteration:
                    del head[k]
                break
        else:
            return False
    return all(not live[wg][k] for wg in (0, 1) for k in ("a", "b"))


GRID = [dict(a_slots=na, b_slots=nb, ngroups=ng, taps=nt, kchunks=kc, planes=pl, items=it)
        for na, nb, ng, nt, kc, pl, it in itertools.product((2, 3, 4), (2, 3, 4), (1, 3), (1, 2, 3), (1, 3), (1, 2),
                                                            (1, 3))]


@pytest.mark.parametrize("lag", [0, 1, 7, 10 ** 6])
def test_rings_always_progress(lag):
    """the ring depths the host uses (paired 3 + 3, unpaired 4 + 4) and every depth >= 2 finish under any lag of one
    warpgroup, from lockstep to one warpgroup running until it blocks"""
    for cfg in GRID:
        assert replay(cfg, lag), f"deadlock: {cfg}, lag {lag}"


def test_model_finds_a_deadlock():
    """one A slot cannot hold a chunk's hi and lo slabs at once: the model must report that, or it checks nothing"""
    cfg = dict(a_slots=1, b_slots=3, ngroups=1, taps=3, kchunks=2, planes=2, items=1)
    assert not replay(cfg, 0)
