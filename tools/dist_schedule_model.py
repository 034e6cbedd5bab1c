"""Discrete-event model of the distributed (block-column-cyclic) Cholesky schedule of fit_dist_impl
(abstractgps.jl_b200/csrc/engine.cu): per rank two in-order streams, CUDA-event edges, one NCCL broadcast per outer panel,
and the one hardware fact that shapes everything -- the persistent int8-slice update kernel holds every SM it was launched
on until it ends, so whatever is enqueued behind it (the next panel's factorisation, the NCCL kernel of the next
broadcast) waits for it.

    python tools/dist_schedule_model.py [--n 65536] [--ranks 8] [--w 512]

It replays the op order of the C++ loop for the default schedule and for AGP_DIST_SCHED=1 (owner defers its rest update
behind the next panel's factorisation; updates leave `reserve` SMs to NCCL), checks that neither order can deadlock,
and prints the modelled makespan.  Durations come from ASSUMED rates, not measurements: update kernel 60 TFLOP/s
fp64-equivalent at full width x a narrow-update efficiency, panel factorisation = 0.28 ms of latency-bound chain + its
flops at 20 TFLOP/s, broadcast at 350 GB/s.  The model is for ranking schedules, not for predicting ms."""
import argparse
import heapq

NSM = 132  # H100 SXM


class Op:
    __slots__ = ("rank", "stream", "name", "dur", "sms", "waits", "records", "coll", "start", "end")

    def __init__(self, rank, stream, name, dur, sms, waits=(), records=(), coll=None):
        self.rank, self.stream, self.name, self.dur, self.sms = rank, stream, name, dur, sms
        self.waits, self.records, self.coll = list(waits), list(records), coll
        self.start = self.end = None


def build(n, R, W, sched2, reserve, eff_narrow):
    lda = n + 128
    nto = n // W
    ops = {(r, st): [] for r in range(R) for st in ("s", "s2")}
    upd_rate, fact_rate, bw = 60e12, 20e12, 350e9

    def t_update(blocks, sms):
        """rank-W update of the local outer blocks `blocks` (global indices): block j takes rows [j W, lda)"""
        if not blocks:
            return 0.0
        flops = sum(2.0 * W * W * (lda - j * W) for j in blocks)
        return flops / (upd_rate * eff_narrow * sms / NSM) + 15e-6

    def t_factor(rows):  # W/128 inner steps of ~70 us latency-bound chain + rows * W^2 flop of TRSM / rank-128 updates
        return (W / 128) * 0.07e-3 + rows * float(W) * W / fact_rate

    for r in range(R):
        S, S2 = ops[(r, "s")], ops[(r, "s2")]
        rest_pending = None
        deferred = None
        for kk in range(nto):
            owner = kk % R
            rows_below = lda - (kk + 1) * W
            if owner == r:
                S.append(Op(r, "s", "factor%d" % kk, t_factor(lda - kk * W), NSM - (reserve if sched2 else 0)))
            if deferred is not None:
                e_fact = ("fact", r, kk)
                S.append(Op(r, "s", "rec_fact%d" % kk, 0.0, 0, records=[e_fact]))
                dk, blocks, e_rest = deferred
                S2.append(Op(r, "s2", "rest%d" % dk, t_update(blocks, NSM - reserve), NSM - reserve,
                             waits=[e_fact], records=[e_rest]))
                deferred = None
            if R > 1:
                S.append(Op(r, "s", "bcast%d" % kk, rows_below * W * 8.0 / bw + 30e-6, reserve if sched2 else 8, coll=("b", kk)))
            if kk == nto - 1:
                break
            waits = [rest_pending] if rest_pending else []
            e_panel, e_rest = ("panel", r, kk), ("rest", r, kk)
            S.append(Op(r, "s", "slice%d" % kk, rows_below * W * 15.0 / 5e12 + 10e-6, NSM, waits=waits, records=[e_panel]))
            # local outer blocks with global index > kk
            loc = [j for j in range(kk + 1, nto) if j % R == r]
            own_next = (kk + 1) % R == r
            if own_next:
                S.append(Op(r, "s", "nextupd%d" % kk, t_update(loc[:1], NSM), NSM))
                loc = loc[1:]
            rest_pending = e_rest
            if sched2 and own_next:
                deferred = (kk, loc, e_rest)
            else:
                S2.append(Op(r, "s2", "rest%d" % kk, t_update(loc, NSM - (reserve if sched2 else 0)),
                             NSM - (reserve if sched2 else 0), waits=[e_panel], records=[e_rest]))
        if rest_pending:
            S.append(Op(r, "s", "join", 0.0, 0, waits=[rest_pending]))
    return ops


def simulate(ops, R):
    """in-order streams; an op starts when it is at the head of its stream, its events are recorded, its SMs are free
    (per rank) and -- for a collective -- every rank has it ready.  Returns (makespan, per-op list) or raises on deadlock."""
    head = {k: 0 for k in ops}
    free = {r: NSM for r in range(R)}
    done_ev = set()
    running = []  # (end, seq, op)
    now, seq = 0.0, 0
    total = sum(len(v) for v in ops.values())
    finished = 0

    def ready(op):
        return all(w in done_ev for w in op.waits) and free[op.rank] >= op.sms

    while finished < total:
        progressed = True
        while progressed:
            progressed = False
            # collectives: all ranks must have the same collective at the head of stream s and be ready
            colls = {}
            for (r, st), lst in ops.items():
                i = head[(r, st)]
                if i < len(lst) and lst[i].start is None and lst[i].coll:
                    colls.setdefault(lst[i].coll, []).append(lst[i])
            for cid, members in colls.items():
                if len(members) == R and all(ready(m) for m in members):
                    for m in members:
                        m.start, m.end = now, now + m.dur
                        free[m.rank] -= m.sms
                        seq += 1
                        heapq.heappush(running, (m.end, seq, m))
                    progressed = True
            for (r, st), lst in ops.items():
                i = head[(r, st)]
                if i < len(lst) and lst[i].start is None and not lst[i].coll and ready(lst[i]):
                    op = lst[i]
                    op.start, op.end = now, now + op.dur
                    free[r] -= op.sms
                    seq += 1
                    heapq.heappush(running, (op.end, seq, op))
                    progressed = True
        if not running:
            stuck = [(k, ops[k][head[k]].name, ops[k][head[k]].waits) for k in ops if head[k] < len(ops[k])]
            raise RuntimeError("deadlock at t=%.3f ms: %s" % (now * 1e3, stuck[:6]))
        end, _, op = heapq.heappop(running)
        now = end
        free[op.rank] += op.sms
        for e in op.records:
            done_ev.add(e)
        head[(op.rank, op.stream)] += 1
        finished += 1
    return now


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--ranks", type=int, default=8)
    ap.add_argument("--w", type=int, default=512)
    ap.add_argument("--reserve", type=int, default=16)
    a = ap.parse_args()
    print("N=%d W=%d: modelled factorisation makespan (ms)" % (a.n, a.w))
    for R in sorted({1, 2, 4, a.ranks}):
        eff = 1.0 if R == 1 else 0.7  # measured: per-rank update kernel time 348 ms at R=8 vs 1916/8 = 240 ms ideal
        base = simulate(build(a.n, R, a.w, False, 0, eff), R)
        line = "  ranks=%d  default order: %7.1f" % (R, base * 1e3)
        if R > 1:
            new = simulate(build(a.n, R, a.w, True, a.reserve, eff), R)
            line += "   AGP_DIST_SCHED=1 (reserve %d SMs): %7.1f  (%.2fx)" % (a.reserve, new * 1e3, base / new)
        print(line)


if __name__ == "__main__":
    main()
