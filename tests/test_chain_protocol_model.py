"""Randomised model of the synchronisation protocol of the persistent convolution kernel (csrc/conv_chain.cu), no GPU.

The kernel's twelve warps talk through mbarriers whose waiters see only a phase PARITY, with three asynchronous agents in
between (cp.async row copies, bulk weight copies, each consumer warpgroup's wgmma groups).  What can go wrong is ordering, not
arithmetic: a producer that passes a parity test one lap early overwrites rows that have not been multiplied, a consumer
that mistakes "lap L-2 filled" for "lap L filled" multiplies stale rows, a role that skips an arrival hangs the CTA.  This
file restates the protocol -- every wait, arrival and slot / phase update of the three roles, in the order the kernel performs
them -- as coroutines over modelled mbarriers, runs it under random schedules (including arbitrarily late completion of
copies and MMAs) and checks that

  * every schedule terminates (no deadlock; a consumer holds the slots of two stages: it frees a stage after wgmma_wait<1>),
  * every MMA reads exactly the row slot and weight slot contents meant for it (stage, sub-tile, item),
  * no row / weight slot is overwritten while an issued MMA still has to read it,
  * a consumer warpgroup's epilogue runs only after all MMAs of its item retired.

The reason every ring slot has a fixed owner is visible here: with ring slots dealt round-robin over the gather
warps (the first version) the same model finds overwritten rows within a few schedules -- the negative control below.
It is a model of the PROTOCOL: what the hardware does inside one instruction (the proxy fences, the swizzle, the descriptors)
is covered by the GPU tests (tests/test_gpu_conv_chain.py: bit-identical repeated launches against the fp64 oracle)."""
import random

import pytest

A_WARPS = 3                     # CH_A_WARPS


class Bar:
    """mbarrier: `count` arrivals (+ outstanding transaction bytes) complete a phase; waiters test a phase parity."""

    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0

    def _maybe_complete(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive(self):
        assert self.pending > 0, "more arrivals than the barrier was initialised for"
        self.pending -= 1
        self._maybe_complete()

    def expect_tx_arrive(self, nbytes):
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._maybe_complete()

    def test(self, parity):                      # mbarrier.try_wait.parity: has the phase of that parity completed?
        return (self.phase & 1) != parity


class Violation(AssertionError):
    pass


class Cta:
    def __init__(self, items, sa, sb, rng, fixed_owners=True, layer_ends=(), a_warps=A_WARPS):
        self.items, self.sa, self.sb, self.rng, self.a_warps = items, sa, sb, rng, a_warps
        self.fixed_owners, self.layer_ends = fixed_owners, set(layer_ends)
        self.fullA = [Bar(1) for _ in range(sa)]            # (32 lane arrivals in the kernel: one modelled completion)
        self.emptyA = [Bar(2) for _ in range(sa)]           # one arrival per consumer warpgroup
        self.fullB = [Bar(1) for _ in range(sb)]
        self.emptyB = [Bar(2) for _ in range(sb)]           # one arrival per consumer warpgroup
        self.slotA = [None] * sa                            # content tags
        self.slotB = [None] * sb
        self.readsA = [0] * sa                              # issued wgmmas (either warpgroup) that still have to read the slot
        self.readsB = [0] * sb
        self.fifo = {}                                      # async agents: name -> list of pending operations (in order)
        self.sync_wait = {}                                 # layer boundary (__syncthreads): role -> layer index reached
        self.n_roles = 1 + a_warps + 2

    # ---- asynchronous agents -------------------------------------------------------------------
    def push(self, agent, op):
        self.fifo.setdefault(agent, []).append(op)

    def run_async(self, agent):
        op = self.fifo[agent].pop(0)
        op()

    # ---- roles (generators: `yield (bar, parity)` = blocked on a wait, `yield None` = scheduling point) ----
    def weights(self):
        b_slot = b_phase = 0
        for it, (nsub, stages) in enumerate(self.items):
            for t in range(stages):
                yield (self.emptyB[b_slot], b_phase ^ 1)
                bar, s, tag = self.fullB[b_slot], b_slot, (it, t)
                bar.expect_tx_arrive(1)

                def land(bar=bar, s=s, tag=tag):
                    if self.readsB[s]:
                        raise Violation(f"weight slot {s} overwritten with {tag} while {self.readsB[s]} MMAs still read {self.slotB[s]}")
                    self.slotB[s] = tag
                    bar.complete_tx(1)
                self.push('bulk', land)
                b_slot += 1
                if b_slot == self.sb:
                    b_slot, b_phase = 0, b_phase ^ 1
                yield None
            yield from self.layer_sync('weights', it)

    def consumer(self, g):
        """chain_item: per stage wait for its slots, issue one wgmma group, wgmma_wait<1>, free the PREVIOUS stage's slots;
        after the item wgmma_wait<0>, free the last stage's slots, epilogue."""
        a_slot = a_phase = b_slot = b_phase = 0
        sa, sb = self.sa, self.sb
        pipe = f'tensor{g}'
        for it, (nsub, stages) in enumerate(self.items):
            acc = dict(done=0)
            prev = None                                        # (row slots, weight slot, group-retired marker) of the last stage
            for t in range(stages):
                rows, phases = [a_slot], [a_phase]
                if nsub == 2:
                    a1, p1 = a_slot + 1, a_phase
                    if a1 >= sa:
                        a1, p1 = a1 - sa, p1 ^ 1
                    rows.append(a1); phases.append(p1)
                yield (self.fullB[b_slot], b_phase)            # (the kernel probes all of them together)
                for a, p in zip(rows, phases):
                    yield (self.fullA[a], p)
                b = b_slot
                for a in rows:
                    self.readsA[a] += 1
                self.readsB[b] += 1
                retired = Bar(1)

                def group(rows=tuple(rows), b=b, it=it, t=t, acc=acc, retired=retired):
                    for s_, a in enumerate(rows):
                        if self.slotA[a] != (it, t, s_):
                            raise Violation(f"consumer {g}: row slot {a} holds {self.slotA[a]}, expected {(it, t, s_)}")
                    if self.slotB[b] != (it, t):
                        raise Violation(f"consumer {g}: weight slot {b} holds {self.slotB[b]}, expected {(it, t)}")
                    for a in rows:
                        self.readsA[a] -= 1
                    self.readsB[b] -= 1
                    acc['done'] += len(rows)
                    retired.arrive()
                self.push(pipe, group)
                if prev is not None:
                    yield (prev[2], 0)                         # wgmma_wait<1>: the previous stage's group has retired
                    for a in prev[0]:
                        self.emptyA[a].arrive()
                    self.emptyB[prev[1]].arrive()
                prev = (rows, b, retired)
                a_slot += nsub
                if a_slot >= sa:
                    a_slot, a_phase = a_slot - sa, a_phase ^ 1
                b_slot += 1
                if b_slot == sb:
                    b_slot, b_phase = 0, b_phase ^ 1
                yield None
            if prev is not None:
                yield (prev[2], 0)                             # wgmma_wait<0>
                for a in prev[0]:
                    self.emptyA[a].arrive()
                self.emptyB[prev[1]].arrive()
            if acc['done'] != stages * nsub:
                raise Violation(f"consumer {g}: epilogue of item {it} after {acc['done']} of {stages * nsub} sub-tile stages")
            yield None                                         # epilogue: registers -> staging -> global
            yield from self.layer_sync(f'consumer{g}', it)

    def gather(self, w):
        sa = self.sa
        g_slot, p_sl, p_lapb, p_par = 0, w, 0, 0
        nxt = w                                              # round-robin variant: my next GLOBAL slot index
        agent = f'copy{w}'
        for it, (nsub, stages) in enumerate(self.items):
            g_end = g_slot + stages * nsub
            while True:
                if self.fixed_owners:                        # ring slot s is always filled by warp s % a_warps
                    if not (w < sa and p_lapb + p_sl < g_end):
                        break
                    sl, par, jl = p_sl, p_par, p_lapb + p_sl - g_slot
                    p_sl += self.a_warps
                    if p_sl >= sa:
                        p_sl, p_lapb, p_par = w, p_lapb + sa, p_par ^ 1
                else:                                        # first version: slots dealt round-robin over the warps
                    if not nxt < g_end:
                        break
                    sl, par, jl = nxt % sa, (nxt // sa) & 1, nxt - g_slot
                    nxt += self.a_warps
                st, s = divmod(jl, nsub)
                yield (self.emptyA[sl], par ^ 1)
                bar, tag = self.fullA[sl], (it, st, s)

                def land(sl=sl, tag=tag):
                    if self.readsA[sl]:
                        raise Violation(f"row slot {sl} overwritten with {tag} while {self.readsA[sl]} MMAs still read {self.slotA[sl]}")
                    self.slotA[sl] = tag
                self.push(agent, land)
                self.push(agent, bar.arrive)                 # cp.async.mbarrier.arrive.noinc: fires when the copies have landed
                yield None
            g_slot = g_end
            yield from self.layer_sync(f'gather{w}', it)

    def layer_sync(self, me, it):
        """__syncthreads() between the layers of a launch: every role waits for every other role here."""
        if it not in self.layer_ends:
            return
        self.sync_wait[me] = it
        while sum(1 for v in self.sync_wait.values() if v >= it) < self.n_roles:
            yield 'sync'

    # ---- scheduler ---------------------------------------------------------------------------------
    def run(self):
        roles = {'weights': self.weights(), 'consumer0': self.consumer(0), 'consumer1': self.consumer(1)}
        roles.update({f'gather{w}': self.gather(w) for w in range(self.a_warps)})
        blocked = {}                                          # role -> (bar, parity) | 'sync'
        steps = 0
        # late completions: with probability `lazy` an asynchronous agent is NOT offered to the scheduler in a round
        lazy = self.rng.choice([0.0, 0.3, 0.7, 0.95])
        while roles:
            steps += 1
            runnable = []
            for name in roles:
                b = blocked.get(name)
                if b is None or b == 'sync' or b[0].test(b[1]):
                    runnable.append(name)
            agents = [a for a, q in self.fifo.items() if q]
            offered = [a for a in agents if self.rng.random() >= lazy]
            only_sync = all(blocked.get(n) == 'sync' for n in runnable)
            if (not runnable or only_sync) and not agents:
                if not runnable:
                    raise Violation(f"deadlock after {steps} steps: " + ", ".join(
                        f"{n} waits parity {b[1]} (phase {b[0].phase})" for n, b in blocked.items() if n in roles and b != 'sync'))
            choices = runnable + (offered or (agents if (not runnable or only_sync) else []))
            pick = self.rng.choice(choices)
            if pick in self.fifo and pick not in roles:
                self.run_async(pick)
                continue
            try:
                y = next(roles[pick])
            except StopIteration:
                del roles[pick]
                blocked.pop(pick, None)
                continue
            if y is None:
                blocked.pop(pick, None)
            else:
                blocked[pick] = y
            if steps > 4_000_000:
                raise Violation("livelock")
        for agent in list(self.fifo):                         # drain: the kernel ends with the last epilogue
            while self.fifo[agent]:
                self.run_async(agent)
        assert not any(self.readsA) and not any(self.readsB)
        return steps


def _items(rng, n, max_stages):
    """a layer list as the kernel sees it: runs of items with one (nsub, stages) shape per layer, odd tails of one sub-tile"""
    items, ends = [], []
    while len(items) < n:
        nsub_max, stages = rng.choice([1, 2, 2]), rng.randint(1, max_stages)
        for _ in range(rng.randint(1, 6)):
            items.append((nsub_max if rng.random() < 0.8 else 1, stages))       # u_end / last-row-tile singles
        ends.append(len(items) - 1)
    return items, ends[:-1]


# the ring shapes osb_conv_chain_launch builds: even row rings of 4..12 slots (4 = the least it accepts: two paired stages),
# 2 to 4 weight slots; the defaults are (10, 3) for N tiles up to 96 columns and (8, 3) for 128
RINGS = [(4, 2), (6, 3), (8, 2), (8, 3), (10, 3), (12, 3), (12, 2), (10, 4)]


@pytest.mark.parametrize('sa,sb', RINGS)
def test_protocol_is_safe_and_live_under_random_schedules(sa, sb):
    for seed in range(40):
        rng = random.Random(1000 * sa + 10 * sb + seed)
        items, ends = _items(rng, rng.randint(3, 14), rng.choice([1, 2, 3, 9, 27]))
        Cta(items, sa, sb, rng, fixed_owners=True, layer_ends=ends).run()


def test_long_single_layer_many_laps():
    rng = random.Random(7)
    Cta([(1, 81)] * 7, 10, 3, rng).run()                      # the level-0 96->96 layer: 27 offsets x 3 channel blocks per item
    Cta([(2, 54)] * 6 + [(1, 54)], 10, 3, rng).run()          # a 64-wide N tile: paired sub-tiles
    Cta([(1, 216)] * 3, 8, 3, rng).run()                      # a 128-wide N tile of a 256-channel layer


def test_model_finds_the_round_robin_bug():
    """Negative control: slots dealt round-robin over the gather warps instead of fixed owners.  A warp then fills slot s on
    lap L and a DIFFERENT warp on lap L+1; nothing orders the two, and once there are at least as many gather warps as ring
    slots the later one can pass the parity test of `emptyA[s]` two phases early (phase L-2 looks like phase L) and overwrite
    rows that were never multiplied -- the defect the first version of the kernel had, with five gather warps on a ring of four
    slots.  The model must catch it there; with fixed owners the same warps and ring are safe."""
    caught = 0
    for seed in range(60):
        rng = random.Random(seed)
        try:
            Cta([(2, 27)] * 8, 4, 2, rng, fixed_owners=False, a_warps=5).run()
        except Violation:
            caught += 1
    assert caught >= 30, f"only {caught} of 60 schedules exposed the known defect"
    for seed in range(20):
        Cta([(2, 27)] * 8, 4, 2, random.Random(seed), fixed_owners=True, a_warps=5).run()
