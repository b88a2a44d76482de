"""Interleaving-level model of the flag / epoch protocol of the fused TP kernels (csrc/gemm_sm90.cu MODE 5 / 6, ops/_fused_impl.py).

Every rank is a coroutine that performs one atomic action per step (a payload write, a flag release, a flag poll, a payload
read); a seeded scheduler picks which rank moves next, so slow / fast rank skews of any size occur.  Checked invariants:

  * a consumer released by ``flag >= epoch`` always reads the payload version of ITS call (never a stale one);
  * a producer never overwrites a parity buffer that some rank has not finished reading from the call two calls ago
    (the "a rank can only be in call n+1 if every peer finished call n-1" argument of DESIGN §2.2);
  * this holds across region re-layouts (larger shapes): a re-layout syncs all ranks and either reuses the region (flags keep
    their old epochs) or maps a fresh one (flags zero).

``reset_epochs=True`` models the round-2 bug (epoch counters restarted at 1 while the reused region still held old epochs): the
model FAILS for it with a stale read, and passes with monotonic epochs — `tests/test_misc_cpu.py` runs both.

``simulate_publish`` models the publish + pull kernels of ``csrc/nvls_coll.cu`` (embedding gather, all-to-all, ``publish`` views).

    python tools/sim_nvls_protocol.py            # 200 random schedules each of the good configurations
"""
from __future__ import annotations

import random
from typing import Dict, List


class StaleRead(AssertionError):
    pass


def simulate(world: int, calls: List[str], blocks: int, relayout_at: int, reuse_region: bool, reset_epochs: bool, seed: int,
             max_steps: int = 2_000_000) -> int:
    """``calls``: sequence of "ag" / "rs".  Returns the number of scheduler steps.  Raises StaleRead on a protocol violation."""
    rnd = random.Random(seed)
    flags: List[Dict] = [dict() for _ in range(world)]          # flags[rank][(kind, src, blk)] = epoch
    data: List[Dict] = [dict() for _ in range(world)]           # data[rank][(kind, parity, src, blk)] = call id that wrote it
    reading: List[Dict] = [dict() for _ in range(world)]        # outstanding reads: key → call id being read by its owner
    progress = [0] * world                                      # call index each rank is executing
    at_barrier = [False] * world

    def rank_prog(r: int):
        epoch = {"ag": 0, "rs": 0}
        for ci, kind in enumerate(calls):
            progress[r] = ci
            if ci == relayout_at:
                at_barrier[r] = True
                while not all(at_barrier[p] or progress[p] > ci for p in range(world)):
                    yield
                if not reuse_region:
                    flags[r].clear()                            # fresh region: this rank's flags are zero again
                if reset_epochs:
                    epoch = {"ag": 0, "rs": 0}
                # second phase of the barrier: nobody proceeds before everybody re-laid out
                at_barrier[r] = "done"
                while not all(at_barrier[p] == "done" or progress[p] > ci for p in range(world)):
                    yield
            epoch[kind] += 1
            e, parity = epoch[kind], epoch[kind] & 1
            if kind == "ag":
                # push my blocks to everyone (multicast store), then release per-(src, blk) flags
                for b in range(blocks):
                    for p in range(world):
                        key = (kind, parity, r, b)
                        if key in reading[p] and reading[p][key] != ci:
                            raise StaleRead(f"rank {r} call {ci} overwrites {key} on rank {p} while call {reading[p][key]} is still reading it")
                        data[p][key] = ci
                        yield
                    for p in range(world):
                        if p != r:
                            flags[p][(kind, r, b)] = max(flags[p].get((kind, r, b), 0), e)
                            yield
                # consume: every remote (src, blk) after its flag
                order = [(s, b) for s in range(world) if s != r for b in range(blocks)]
                rnd.shuffle(order)
                for s, b in order:
                    while flags[r].get((kind, s, b), 0) < e:
                        yield
                    key = (kind, parity, s, b)
                    reading[r][key] = ci
                    yield
                    if data[r].get(key) != ci:
                        raise StaleRead(f"rank {r} call {ci} ({kind}) read version {data[r].get(key)} of {key}")
                    yield
                    del reading[r][key]
            else:
                # partial tiles into MY buffer for every owner's blocks, flag the owner per finished block
                for owner in range(world):
                    for b in range(blocks):
                        key = (kind, parity, owner, b)              # lives in data[r]: my partial of owner's block b
                        for q in range(world):
                            if ("pull", r, key) in reading[q] and reading[q][("pull", r, key)] != ci:
                                raise StaleRead(f"rank {r} call {ci} overwrites its partial {key} while rank {q} still pulls call {reading[q][('pull', r, key)]}")
                        data[r][key] = ci
                        yield
                        flags[owner][(kind, r, b)] = max(flags[owner].get((kind, r, b), 0), e)
                        yield
                for b in range(blocks):
                    for s in range(world):
                        while flags[r].get((kind, s, b), 0) < e:
                            yield
                    for s in range(world):                          # pull all ranks' partials of my block b
                        key = (kind, parity, r, b)
                        reading[r][("pull", s, key)] = ci
                        yield
                        if data[s].get(key) != ci:
                            raise StaleRead(f"rank {r} call {ci} (rs) pulled version {data[s].get(key)} of rank {s}'s {key}")
                        del reading[r][("pull", s, key)]
        progress[r] = len(calls)

    progs = [rank_prog(r) for r in range(world)]
    alive = list(range(world))
    steps = 0
    while alive:
        r = rnd.choice(alive) if rnd.random() < 0.7 else alive[0]          # bias towards one rank running far ahead sometimes
        try:
            next(progs[r])
        except StopIteration:
            alive.remove(r)
        steps += 1
        if steps > max_steps:
            raise RuntimeError("protocol model did not terminate (deadlock?)")
    return steps


def simulate_publish(world: int, calls: int, ctas: int, seed: int, single_buffer: bool = False, reads_outlive: int = 0,
                     max_steps: int = 2_000_000) -> int:
    """Model of ``nvls_publish_kernel`` + readers (csrc/nvls_coll.cu; ops.nvls.publish / embedding_gather / all_to_all /
    pull_attention): per call every rank's CTA ``c`` copies slice ``c`` of its buffer into half ``call & 1`` of its OWN slot,
    bumps counter ``c`` on every rank, waits until counter ``c`` shows ``world`` arrivals of this call; after its LAST CTA
    passed, the rank reads every peer's slot (any slice) and only then starts the next call.

    Checked: a reader only ever sees the version of its own call.  ``single_buffer=True`` (no parity halves) must FAIL — a
    fast rank overwrites its slot while a slow peer still reads the previous call.  ``reads_outlive=k`` models views that are
    still read after the rank has passed the barrier of call ``n + k``: already k = 1 FAILS (once a rank has arrived at call
    n+1 its peers may run ahead into call n+2 and rewrite half ``n & 1``) — which is why ``ops.nvls.publish`` promises its views
    only until the caller's NEXT publish and ``pull_attention`` re-publishes K/V in its backward."""
    rnd = random.Random(seed)
    slot = [[[-1] * ctas for _ in range(2)] for _ in range(world)]      # slot[rank][half][slice] = call id that wrote it
    counter = [[0] * ctas for _ in range(world)]                         # counter[rank][cta]: arrivals seen by that rank
    pending: List[List] = [[] for _ in range(world)]                     # (due_call, src, half, slice, expected version)

    def check(r, src, half, sl, want, when):
        got = slot[src][half][sl]
        if got != want:
            raise StaleRead(f"rank {r} at call {when} read version {got} of rank {src} half {half} slice {sl}, expected {want}")

    def rank_prog(r: int):
        for ci in range(calls):
            half = 0 if single_buffer else ci & 1
            order = list(range(ctas))
            rnd.shuffle(order)                                           # CTAs of one rank run in any order
            for c in order:
                slot[r][half][c] = ci                                    # copy my slice
                yield
                for p in range(world):                                   # arrive on every rank's counter c
                    counter[p][c] += 1
                    yield
            for c in order:                                              # ... and wait for this call's arrivals (kernel end = all CTAs)
                while counter[r][c] < (ci + 1) * world:
                    yield
            # late readers of earlier calls' views
            for item in [x for x in pending[r] if x[0] == ci]:
                check(r, item[1], item[2], item[3], item[4], ci)
                yield
            pending[r][:] = [x for x in pending[r] if x[0] != ci]
            reads = [(s, c) for s in range(world) for c in range(ctas)]
            rnd.shuffle(reads)
            for s, c in reads:                                           # pull kernels read any slice of any peer
                check(r, s, half, c, ci, ci)
                if reads_outlive and ci + reads_outlive < calls:
                    pending[r].append((ci + reads_outlive, s, half, c, ci))
                yield

    progs = [rank_prog(r) for r in range(world)]
    alive = list(range(world))
    steps = 0
    while alive:
        r = rnd.choice(alive)
        try:
            next(progs[r])
        except StopIteration:
            alive.remove(r)
        steps += 1
        if steps > max_steps:
            raise RuntimeError("publish protocol model did not terminate (deadlock?)")
    return steps


def main() -> None:
    rnd = random.Random(0)
    n = 0
    for seed in range(200):
        world = rnd.choice([2, 3, 4])
        calls = [rnd.choice(["ag", "rs"]) for _ in range(rnd.randint(3, 9))]
        at = rnd.randint(1, len(calls) - 1)
        for reuse, reset in ((True, False), (False, False), (False, True)):
            simulate(world, calls, rnd.choice([1, 2]), at, reuse, reset, seed)
            n += 1
    print(f"nvls protocol model: {n} schedules ok")
    m = 0
    for seed in range(200):
        simulate_publish(rnd.choice([2, 3, 4]), rnd.randint(2, 7), rnd.choice([1, 2, 3]), seed)
        m += 1
    print(f"publish / pull protocol model: {m} schedules ok")


if __name__ == "__main__":
    main()
