#!/usr/bin/env python
"""Discrete-event model of the synchronisation protocol of a warp-specialised variant of the fused point kernel: a CTA pair
sharing tensor-memory accumulators, weight-producer warps, one or two MMA issuer warps, two epilogue groups and a front end.
It is not the protocol of the shipped kernel (disn_b200/csrc/point_tc.cu, two consumer warpgroups with register
accumulators); it is kept as a checker for that deeper pipeline organisation.

Why: on the GPU a protocol bug is a 4-second trap or silent corruption and costs a scarce GPU run; most of them (dead-
locks, a parity wait by an agent that skipped a phase, a ring slot overwritten before it was consumed, an accumulator
overwritten while it is still being drained) are properties of the *protocol*, not of the hardware.  This model runs
the agents as Python generators over mbarrier objects with the hardware's semantics (arrival counts, phases, parity waits
that can alias), under randomised operation latencies, and checks:
  * no deadlock (every agent terminates);
  * every successful parity wait observed exactly the phase the agent meant (no aliasing, no overrun);
  * every MMA reads the weight stage / activation slice it expects (ring contents are versioned);
  * no accumulator region is written while an overlapping older accumulator still has undrained slices.
One CTA of the pair is modelled (arrival counts that come from both CTAs are halved; the peer adds latency only).

The operation costs in PARAMS are nominal cycle counts, not measurements; `report()` prints modelled cycles per tile and
the per-agent blocked time, and `--set key=value` / `--mode` explore what-ifs (ring depths, operand mode, ...).

    python tools/tc_protocol_sim.py [--tiles N] [--schedules N] [--mode f16f8|bf16x3] [--set key=value ...] [--report]
"""
import argparse
import heapq
import random

SLICES = {0: 1, 1: 4, 2: 8, 3: 8}          # K slices per tensor-core layer (L0..L3 = fold1/conv2 .. fold2/conv2)
NNB = {0: 1, 1: 2, 2: 2, 3: 1}
XS = 20                                     # ring slices per stream (X3: 4, X4: 8, X5: 8); X2 has its own slot

PARAMS = dict(
    NW=3, NX=3, NG=2,
    x2_in_ring=0,      # 1 = fold1/conv1's output goes through the activation ring (staged by epilogue group 0 from the points
                       #     the front end publishes), freeing the dedicated 16 KB slot for a fourth weight stage
    split_wfull=0,     # issuers=2 only: 1 = one 'stage landed' barrier per (issuer, slot), signalled according to the static
                       #     stage -> issuer map, so that an issuer only ever waits on barriers whose every phase is its own
    issuers=1,         # 2 = the dual-issuer variant: one MMA warp per N-block,
                       #     producers with fixed slot ownership that do not wait for the data, peer relay warp
    op=100,            # an mbarrier try_wait that succeeds at once / an arrive, on a busy SM
    commit=150,        # tcgen05.commit
    wake=150,          # arrival -> blocked waiter running again (poll + wake-up), incl. the remote arrive of the peer CTA
    mma_issue=112,     # 8 MMA instructions of one stage
    mma_exec=512,      # tensor-pipe time of one stage (8 x 64 cycles); 768 for bf16x3 (12 MMAs)
    stage_misc=200,    # fences, elect, descriptor/ring bookkeeping per stage
    w_copy=600,        # bulk copy L2 -> smem (32 KB as 2 x 16 KB) issue -> complete_tx
    w_relay=150,       # peer CTA observes its half and arrives on the leader's barrier
    prod_issue=100,    # producer: slot release observed -> copies issued
    drain_pre=250,     # tcgen05.ld + bias (+ gather add) + ReLU
    drain_post=800,    # operand split, 8 x 16 B stores, proxy fence, arrive
    final_ld=300,      # one 32-column slice of the last layer (ld + dot product)
    gather_slice=1700, # front end: 4-tap gather of 64 points x 64 channels
    x2_stage=400, points=500,
    jitter=0.25,
)


def acc_cols(layer, q):
    """[start, end) TMEM columns of the accumulator written by `layer` of a stream with parity q (acc_col() + width)."""
    base = (128 if layer == 0 else (0 if layer == 2 else 256)) ^ (q << 8)
    return base, base + (128 if layer in (0, 3) else 256)


class Bar:
    def __init__(self, name, count):
        self.name, self.count, self.pending, self.phase = name, count, count, 0
        self.waiters = []

    def parity_done(self, parity):          # mbarrier.try_wait.parity semantics
        return (self.phase & 1) != parity


class Sim:
    def __init__(self, tiles, seed, mutate=None, params=None):
        self.mutate = mutate
        self.P = dict(PARAMS)
        if params:
            self.P.update(params)
        self.rng = random.Random(seed)
        self.t, self.q, self.n, self.progress_t = 0, [], 0, 0
        self.T, self.S = tiles, 2 * tiles
        self.mma_tail = 0                   # completion time of the last MMA in the tensor-pipe FIFO
        self.mma_busy = 0
        NW, NX, NG = self.P["NW"], self.P["NX"], self.P["NG"]
        B = Bar
        self.wfull = [B("wfull%d" % i, 1) for i in range(NW)]      # {expect_tx arrival + bytes}: one event here
        self.wempty = [B("wempty%d" % i, 1) for i in range(NW)]
        self.wfull_i = [[B("wfull%c%d" % ("AB"[w], i), 1) for i in range(NW)] for w in range(2)]
        self.wuse = [[0] * NW for _ in range(2)]      # per issuer: uses of each slot so far
        self.xfull = [B("xfull%d" % i, 1) for i in range(NX)]       # per group-slice (4 warps x 2 CTAs in hardware)
        self.xempty = [B("xempty%d" % i, self.P["issuers"]) for i in range(NX)]
        self.x2full, self.x2empty = B("x2full", 1), B("x2empty", 1)
        self.pfull = [B("pfull%d" % i, 1) for i in range(2)]          # points of tile parity i published by the front end
        self.points = [None, None]
        self.gfull = [B("gfull%d" % i, 1) for i in range(NG)]
        self.gempty = [B("gempty%d" % i, 1) for i in range(NG)]
        self.acc_full = [[B("acc%d_%d" % (l, nb), 1) for nb in range(2)] for l in range(4)]
        self.acc5_free = B("acc5_free", 2)                          # both epilogue groups
        self.w_slot, self.x_slot, self.x2_slot, self.g_slot = [None] * NW, [None] * NX, None, [None] * NG
        self.live = []                       # accumulator N-blocks with undrained slices: [cols, remaining, tag]
        self.blocked = {}
        self.stats = {}                      # (agent, barrier class) -> blocked cycles

    # ---- event loop -------------------------------------------------------------------------------
    def d(self, key, scale=1.0):
        v = self.P[key] * scale
        j = self.P["jitter"]
        return max(1, int(v * self.rng.uniform(1 - j, 1 + j)))

    def at(self, dt, fn):
        self.n += 1
        heapq.heappush(self.q, (self.t + dt, self.n, fn))

    def arrive(self, bar):
        bar.pending -= 1
        assert bar.pending >= 0, "too many arrivals on " + bar.name
        if bar.pending == 0:
            bar.phase += 1
            bar.pending = bar.count
            ws, bar.waiters = bar.waiters, []
            for w in ws:
                w()

    def spawn(self, name, gen):
        def step(val=None):
            self.progress_t = self.t
            try:
                op = gen.send(val)
            except StopIteration:
                self.blocked.pop(name, None)
                return
            kind = op[0]
            if kind == "delay":
                self.at(op[1], step)
            elif kind == "wait":
                _, bar, parity, want = op
                t0 = self.t
                cls = bar.name.rstrip("0123456789_")

                def check(first=True):
                    if bar.parity_done(parity):
                        assert bar.phase == want + 1, "%s: wait on %s meant phase %d but the barrier has completed %d" % (
                            name, bar.name, want, bar.phase)
                        self.blocked.pop(name, None)
                        cost = self.d("op") if first else self.d("wake")
                        self.stats[(name, cls)] = self.stats.get((name, cls), 0) + (self.t - t0) + cost
                        self.at(cost, step)
                    else:
                        self.blocked[name] = (bar.name, want, bar.phase)
                        bar.waiters.append(lambda: check(False))
                check()
            else:
                raise ValueError(kind)
        self.blocked[name] = ("start", 0, 0)
        self.at(0, step)

    def run(self):
        while self.q:
            self.t, _, fn = heapq.heappop(self.q)
            fn()
        assert not self.blocked, "deadlock: " + repr(self.blocked)

    # ---- tensor pipe ------------------------------------------------------------------------------
    def issue_mmas(self, dur):
        self.mma_tail = max(self.mma_tail, self.t) + dur
        self.mma_busy += dur

    def commit(self, bar):                   # tcgen05.commit: arrive when everything issued so far has retired
        self.at(max(0, self.mma_tail - self.t) + self.d("op", 0.5), lambda: self.arrive(bar))

    # ---- agents -----------------------------------------------------------------------------------
    def seq_of(self, sn, kind, t=0):
        """index of an activation slice in the ring's production/consumption order; kind: 2 (fold1/conv1 output of stream sn,
        only with x2_in_ring), 3, 4, 5 (outputs of tensor-core layers L0, L1, L2 of stream sn)"""
        if not self.P["x2_in_ring"]:
            return sn * XS + {3: 0, 4: 4, 5: 12}[kind] + t
        if kind == 2:
            return 0 if sn == 0 else 1 + 21 * (sn - 1) + 12
        base = 1 + 21 * sn
        if kind == 5:
            return base + 12 + (1 if sn + 1 < self.S else 0) + t
        return base + {3: 0, 4: 4}[kind] + t

    def build_order(self):
        """the MMA warp's issue order == the weight stages' consumption order (streams skewed by one layer)"""
        order = []

        def layer(sn, l):
            for t in range(SLICES[l]):
                for nb in range(NNB[l]):
                    order.append((sn, l, t, nb))
        if self.S:
            layer(0, 0)
        for sn in range(self.S):
            layer(sn, 1)
            layer(sn, 2)
            if sn + 1 < self.S:
                layer(sn + 1, 0)
            layer(sn, 3)
        self.order = order

    def producer(self, pw):
        NW = self.P["NW"]
        g = pw
        while g < len(self.order):
            use = g // NW
            if self.mutate != "no_wempty_wait":
                yield ("wait", self.wempty[pw], (use & 1) ^ 1, use - 1)
            yield ("delay", self.d("prod_issue"))

            def land(g=g, pw=pw):
                self.w_slot[pw] = g
                self.arrive(self.wfull[pw])
            self.at(self.d("w_copy") + self.d("w_relay"), land)
            yield ("wait", self.wfull[pw], use & 1, use)          # relay (peer) / re-arm expect_tx (leader)
            yield ("delay", self.d("op"))
            g += NW

    def producer_owned(self, slots):
        """dual-issuer variant: this warp owns `slots` (every phase of their barriers is observed by it alone) and never
        waits for the data; arrival is observed by the issuers (leader) / relayed by the peer's warp 1"""
        NW = self.P["NW"]
        for g in range(len(self.order)):
            slot = g % NW
            if slot not in slots:
                continue
            use = g // NW
            yield ("wait", self.wempty[slot], (use & 1) ^ 1, use - 1)
            yield ("delay", self.d("prod_issue") + self.d("op"))

            def land(g=g, slot=slot):
                self.w_slot[slot] = g
                if self.P["split_wfull"]:
                    sn_, l_, t_, nb_ = self.order[g]
                    self.arrive(self.wfull_i[nb_ if NNB[l_] == 2 else 0][slot])
                else:
                    self.arrive(self.wfull[slot])
            self.at(self.d("w_copy") + self.d("w_relay"), land)

    def mma(self, which=0):
        NW, NX = self.P["NW"], self.P["NX"]
        dual = self.P["issuers"] == 2
        g = 0
        xseq = 0
        for (sn, l, t, nb) in self.order:
            q = sn & 1
            mine = (not dual) or (nb == which if NNB[l] == 2 else which == 0)
            if dual and not mine:                        # the other issuer's stage
                ring = l != 0 or self.P["x2_in_ring"]
                if nb == 0 and ring:                     # still observe the activation slice (keeps the two in step)
                    slot = xseq % NX
                    yield ("wait", self.xfull[slot], (xseq // NX) & 1, xseq // NX)
                if t == 0 and nb == 0 and l == 2 and sn > 0:
                    yield ("wait", self.acc5_free, (sn - 1) & 1, sn - 1)
                if self.mutate != "dual_skip_phases" and not self.P["split_wfull"]:
                    yield ("wait", self.wfull[g % NW], (g // NW) & 1, g // NW)   # observe every phase of the slot
                if NNB[l] == 1 and ring:                 # nothing to issue on this slice: release it right away
                    self.arrive(self.xempty[xseq % NX])
                    yield ("delay", self.d("commit"))
                if nb == NNB[l] - 1 and ring:
                    xseq += 1
                g += 1
                continue
            if t == 0 and nb == (which if (dual and NNB[l] == 2) else 0):
                if l == 2 and sn > 0 and self.mutate != "no_acc5_wait":
                    yield ("wait", self.acc5_free, (sn - 1) & 1, sn - 1)
                cols = acc_cols(l, q)
                for c, rem, tag in self.live:           # write-after-read hazard on TMEM
                    assert rem == 0 or c[1] <= cols[0] or cols[1] <= c[0], \
                        "L%d of stream %d overwrites %s with %d undrained slices" % (l, sn, tag, rem)
                self.live = [e for e in self.live if e[1] > 0]
            if nb == 0 or (dual and which == 1):         # activation slice (first stage of the slice for this issuer)
                if l == 0 and not self.P["x2_in_ring"]:
                    yield ("wait", self.x2full, sn & 1, sn)
                    assert self.x2_slot == sn, "X2 slot holds stream %r, wanted %d" % (self.x2_slot, sn)
                else:
                    slot = xseq % NX
                    yield ("wait", self.xfull[slot], (xseq // NX) & 1, xseq // NX)
                    want = self.seq_of(sn, 2 + l, t)
                    assert want == xseq, "ring order: issuer at %d, slice is %d" % (xseq, want)
                    assert self.x_slot[slot] == want, "X slot %d holds %r, wanted %d" % (slot, self.x_slot[slot], want)
            st = g % NW
            if dual and self.P["split_wfull"]:
                u = self.wuse[which][st]
                self.wuse[which][st] += 1
                yield ("wait", self.wfull_i[which][st], u & 1, u)
            else:
                yield ("wait", self.wfull[st], (g // NW) & 1, g // NW)
            assert self.w_slot[st] == g, "W slot %d holds stage %r, wanted %d" % (st, self.w_slot[st], g)
            yield ("delay", self.d("stage_misc") + self.d("mma_issue"))
            self.issue_mmas(self.P["mma_exec"])
            ncommit = 1
            self.commit(self.wempty[st])
            if t == SLICES[l] - 1:                       # this N-block (128 columns = 4 drain slices) is final
                self.commit(self.acc_full[l][nb])
                ncommit += 1
                c0 = acc_cols(l, q)[0] + 128 * nb
                self.at(max(0, self.mma_tail - self.t),
                        lambda c=(c0, c0 + 128), tag="acc of L%d/%d stream %d" % (l, nb, sn): self.live.append([c, 4, tag]))
            if nb == NNB[l] - 1 or dual:                 # dual: each issuer releases the slice after its own stage
                ncommit += 1
                if l == 0 and not self.P["x2_in_ring"]:
                    self.commit(self.x2empty)
                else:
                    self.commit(self.xempty[xseq % NX])
            if nb == NNB[l] - 1 and (l != 0 or self.P["x2_in_ring"]):
                xseq += 1
            yield ("delay", ncommit * self.d("commit"))
            g += 1

    def drained(self, l, q, t):              # 32-column slice t of the accumulator written by layer l was read
        c0 = acc_cols(l, q)[0] + 128 * (t // 4)
        cols = (c0, c0 + 128)
        for e in self.live:
            if e[0] == cols and e[1] > 0:
                e[1] -= 1
                return
        raise AssertionError("drain of an accumulator that is not complete: L%d parity %d" % (l, q))

    def epilogue(self, eg):
        NX = self.P["NX"]
        gcount = 0

        def drain(sn, l_acc, t, seq, gather):
            """read slice t of the accumulator written by layer l_acc, write activation slice `seq`"""
            nonlocal gcount
            yield ("delay", self.d("drain_pre"))
            if gather:
                gs = t % self.P["NG"]
                yield ("wait", self.gfull[gs], (gcount_of(sn, t) // 1) & 1, gcount_of(sn, t))
                assert self.g_slot[gs] == (sn >> 1) * 8 + t, "gather slot %d holds %r" % (gs, self.g_slot[gs])
            self.drained(l_acc, sn & 1, t)
            slot = seq % NX
            if self.mutate != "no_xempty_wait":
                yield ("wait", self.xempty[slot], ((seq // NX) & 1) ^ 1, seq // NX - 1)
            yield ("delay", self.d("drain_post"))
            self.x_slot[slot] = seq
            self.arrive(self.xfull[slot])
            if gather:
                self.arrive(self.gempty[t % self.P["NG"]])

        def gcount_of(sn, t):                # phase index of the gather slot this slice uses
            return ((sn >> 1) * 8 + t) // self.P["NG"]

        def x3(sn):
            for t in range(eg, 4, 2):
                if t == eg:
                    yield ("wait", self.acc_full[0][0], sn & 1, sn)
                yield from drain(sn, 0, t, self.seq_of(sn, 3, t), False)

        def x2(sn):                          # fold1/conv1 of stream sn from the published points (group 0 only)
            tile = sn >> 1
            yield ("wait", self.pfull[tile & 1], (tile >> 1) & 1, tile >> 1)
            assert self.points[tile & 1] == tile, "points buffer holds tile %r, wanted %d" % (self.points[tile & 1], tile)
            seq = self.seq_of(sn, 2)
            slot = seq % NX
            yield ("wait", self.xempty[slot], ((seq // NX) & 1) ^ 1, seq // NX - 1)
            yield ("delay", self.d("x2_stage"))
            self.x_slot[slot] = seq
            self.arrive(self.xfull[slot])
        ring2 = self.P["x2_in_ring"] and eg == 0
        if self.S:
            if ring2:
                yield from x2(0)
            yield from x3(0)
        for sn in range(self.S):
            for l_acc, off in ((1, 4), (2, 12)):
                for t in range(eg, 8, 2):
                    if t == eg and self.mutate != "no_acc_wait":
                        yield ("wait", self.acc_full[l_acc][0], sn & 1, sn)
                    if t == eg + 4:
                        yield ("wait", self.acc_full[l_acc][1], sn & 1, sn)
                    yield from drain(sn, l_acc, t, self.seq_of(sn, 3 + l_acc, t), l_acc == 2 and (sn & 1) == 1)
                if l_acc == 1 and ring2 and sn + 1 < self.S:
                    yield from x2(sn + 1)         # ring order: ... X4_n, X2_{n+1}, X5_n ...
            if sn + 1 < self.S and self.mutate != "x3_after_final":
                yield from x3(sn + 1)
            yield ("wait", self.acc_full[3][0], sn & 1, sn)
            for t in (2 * eg, 2 * eg + 1):
                yield ("delay", self.d("final_ld"))
                self.drained(3, sn & 1, t)
            self.arrive(self.acc5_free)
            if sn + 1 < self.S and self.mutate == "x3_after_final":
                yield from x3(sn + 1)

    def front_end(self):
        NG = self.P["NG"]

        def stage_x2(use):
            yield ("wait", self.x2empty, (use & 1) ^ 1, use - 1)
            yield ("delay", self.d("x2_stage"))
            self.x2_slot = use
            self.arrive(self.x2full)
        def publish(tile):
            yield ("delay", self.d("points"))
            self.points[tile & 1] = tile
            self.arrive(self.pfull[tile & 1])
        if self.P["x2_in_ring"]:
            if self.T:
                yield from publish(0)
        elif self.T:
            yield ("delay", self.d("points"))
            yield from stage_x2(0)
        for it in range(self.T):
            if self.P["x2_in_ring"]:
                if it + 1 < self.T:
                    yield from publish(it + 1)
            else:
                yield from stage_x2(2 * it + 1)
                if it + 1 < self.T:
                    yield ("delay", self.d("points"))
                    yield from stage_x2(2 * it + 2)
            for t in range(8):
                gsq = it * 8 + t
                gs = gsq % NG
                yield ("wait", self.gempty[gs], ((gsq // NG) & 1) ^ 1, gsq // NG - 1)
                yield ("delay", self.d("gather_slice"))
                self.g_slot[gs] = gsq
                self.arrive(self.gfull[gs])


def simulate(tiles=3, seed=0, mutate=None, params=None, want_sim=False):
    """mutate: None (the kernel's protocol); 'no_xempty_wait', 'no_wempty_wait', 'no_acc_wait' are deliberately broken variants
    (tests/test_protocol_cpu.py uses them to show that the checks bite), and 'dual_skip_phases' (issuers=2 where an issuer only
    waits for its own stages -- the aliasing bug of the first dual-issuer attempt); 'x3_after_final' (the un-skewed epilogue order) and
    'no_acc5_wait' are legal-but-slower / redundant-in-this-model variants."""
    s = Sim(tiles, seed, mutate, params)
    assert s.P["NG"] == 2 or s.P["NG"] % 2 == 0, "gather ring depth must be even (slice parity <-> epilogue group)"
    s.build_order()
    if s.P["issuers"] == 2:
        assert s.P["NW"] >= 3
        s.spawn("producer0", s.producer_owned({0}))
        s.spawn("producer1", s.producer_owned(set(range(1, s.P["NW"]))))
        s.spawn("mma", s.mma(0))
        s.spawn("mmaB", s.mma(1))
    else:
        for pw in range(s.P["NW"]):
            s.spawn("producer%d" % pw, s.producer(pw))
        s.spawn("mma", s.mma())
    for eg in range(2):
        s.spawn("epilogue%d" % eg, s.epilogue(eg))
    s.spawn("front", s.front_end())
    s.run()
    return s if want_sim else s.t


def report(tiles, schedules, params):
    tot, busy, stats = 0, 0, {}
    for seed in range(schedules):
        s = simulate(tiles, seed, params=params, want_sim=True)
        tot += s.t
        busy += s.mma_busy
        for k, v in s.stats.items():
            stats[k] = stats.get(k, 0) + v
    n = tiles * schedules
    print("cycles/tile %.0f   tensor pipe busy %.0f (%.0f %%)" % (tot / n, busy / n, 100.0 * busy / tot))
    for (agent, cls), v in sorted(stats.items()):
        if agent in ("mma", "epilogue0", "front", "producer0"):
            print("  %-10s blocked on %-9s %7.0f cycles/tile" % (agent, cls, v / n))


if __name__ == "__main__":
    import signal
    signal.signal(signal.SIGPIPE, signal.SIG_DFL)
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=6)
    ap.add_argument("--schedules", type=int, default=20)
    ap.add_argument("--mode", default="f16f8", choices=["f16f8", "bf16x3"])
    ap.add_argument("--set", action="append", default=[], help="key=value overrides of PARAMS")
    ap.add_argument("--report", action="store_true")
    a = ap.parse_args()
    prm = {}
    if a.mode == "bf16x3":
        prm.update(mma_exec=768, mma_issue=168)
    for kv in a.set:
        k, v = kv.split("=")
        prm[k] = type(PARAMS[k])(float(v))
    if a.report:
        report(a.tiles, a.schedules, prm)
    else:
        ts = [simulate(a.tiles, seed, params=prm) for seed in range(a.schedules)]
        print("%d schedules x %d tiles: no deadlock, no aliased wait, no ring/TMEM hazard; model time %d..%d cycles/tile"
              % (a.schedules, a.tiles, min(ts) // a.tiles, max(ts) // a.tiles))
