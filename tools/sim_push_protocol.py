"""Event-level model of tma_push_stream (the all-gather pusher protocol of the fused TP GEMMs): random load/store latencies and item-ready times; asserts that a
smem stage is never reloaded before its previous store has been read out, that no chunk is stored before it is loaded or before
its item is ready, and that an item's flag is published only after all of its stores have completed, in order."""
import random
def simulate(n_items, cpi, NST, ready_times, seed):
    rnd = random.Random(seed)
    t = 0.0
    total = n_items * cpi
    load_done = {}      # g -> time load completes
    store_read_done = {}; store_done = {}   # g -> times
    stage_owner = {}    # stage -> chunk currently (being) loaded/held
    published = []
    next_flag = 0; issued = 0; ready_upto = 0
    committed = []      # list of g in commit order
    def wait_group(N, read):
        nonlocal t
        # all but the most recent N groups must be complete
        older = committed[:-N] if N > 0 else committed[:]
        for g in older:
            t = max(t, (store_read_done if read else store_done)[g])
    def publish_upto(k_end):
        nonlocal next_flag
        while next_flag < k_end:
            k = next_flag
            for c in range(cpi):
                g = k * cpi + c
                assert g in store_done and store_done[g] <= t + 1e-9, ("flag before store complete", k, g, t)
            published.append(k); next_flag += 1
    def is_ready(k): return ready_times[k] <= t
    for g in range(total):
        while issued < total and issued < g + NST - 1 + (1 if g == 0 else 0):
            k = issued // cpi
            if k >= ready_upto:
                if not is_ready(k):
                    if issued > g: break
                    wait_group(0, False); publish_upto(g // cpi)
                    t = max(t, ready_times[k])
                ready_upto = k + 1
            if issued >= NST: wait_group(1, True)
            st = issued % NST
            if st in stage_owner:
                prev = stage_owner[st]
                assert prev in store_read_done and store_read_done[prev] <= t + 1e-9, ("stage reuse before read done", st, prev, issued, t)
            assert ready_times[issued // cpi] <= t + 1e-9
            stage_owner[st] = issued
            load_done[issued] = t + rnd.uniform(0.5, 2.0)
            issued += 1
            t += 0.01
        assert g in load_done, ("store of unloaded chunk", g)
        t = max(t, load_done[g])
        # store
        rd = t + rnd.uniform(0.2, 1.0)
        prev_done = store_done[committed[-1]] if committed else 0
        store_read_done[g] = rd
        store_done[g] = max(rd + rnd.uniform(0.5, 3.0), prev_done)   # in-order completion
        committed.append(g)
        t += 0.01
        wait_group(NST, False)
        done_upto = g - NST
        if done_upto >= 0: publish_upto((done_upto + 1) // cpi)
    wait_group(0, False); publish_upto(n_items)
    assert published == list(range(n_items))
    return t
for seed in range(300):
    rnd = random.Random(1000 + seed)
    n_items = rnd.randint(1, 6); cpi = rnd.choice([1, 2, 5, 32]); NST = rnd.choice([2, 3, 6])
    ready = sorted(rnd.uniform(0, 40) if rnd.random() < 0.6 else 0.0 for _ in range(n_items))
    simulate(n_items, cpi, NST, ready, seed)
    simulate(n_items, cpi, NST, [0.0] * n_items, seed)
print("protocol simulation ok")
