"""The Cholesky factorisation's schedule (potrf.cu potrf_plan, exported as lb_debug_potrf_plan) checked on the host: every
tile receives each panel exactly once in ascending contiguous ranges, every pass reads only panels whose chain is ordered
before it, no two unordered operations touch the same block column, and the main stream carries exactly the flops bench.py
counts for the trailing update.  No device is needed: the plan is host code."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MAX_COLS = 64                   # SYRK_MAX_COLS
REC = 6 + MAX_COLS              # {op, stream, arg, j0, nc, kend, kb[MAX_COLS]}
POP_PAIR, POP_UPDATE, POP_RECORD, POP_WAIT = 0, 1, 2, 3
MAIN, SIDE = 0, 1
NB = 128


def plan(lib, T, sms):
    n = lib.lb_debug_potrf_plan(T, sms, None, 0)
    assert n > 0, n
    buf = np.zeros((n, REC), dtype=np.int32)
    assert lib.lb_debug_potrf_plan(T, sms, buf.ctypes.data_as(C.c_void_p), n) == n
    return buf


def check_plan(ops, T):
    n = len(ops)
    anc = [0] * n                      # bit m of anc[i]: op m is ordered before (or is) op i
    last = {MAIN: None, SIDE: None}
    recorded = {}
    writes, reads = [0] * n, [0] * n   # block-column masks
    done = {}                          # panel p -> op that finalises it (its pair)
    contrib = {j: [] for j in range(T)}  # column j -> [(op, first panel, end panel, stream)]
    main_flops = 0.0
    for i, r in enumerate(ops):
        op, st, arg, j0, nc, kend = (int(v) for v in r[:6])
        kb = [int(v) for v in r[6:6 + nc]]
        assert st in (MAIN, SIDE)
        a = 1 << i
        if last[st] is not None:
            a |= anc[last[st]]
        if op == POP_WAIT:
            assert arg in recorded, f"op {i}: wait on event {arg} before any record"
            a |= anc[recorded[arg]]
        anc[i] = a
        last[st] = i
        if op == POP_RECORD:
            assert 0 <= arg <= 5
            recorded[arg] = i
        elif op == POP_PAIR:
            k = arg
            assert st == SIDE and k % 2 == 0 and 0 <= k < T
            cols = [k] + ([k + 1] if k + 1 < T else [])
            for j in cols:
                # column j is final before the chain factors it: panels 0 .. k-1 ordered before the pair (panel k of
                # column k+1 is applied inside it)
                assert all((a >> c[0]) & 1 for c in contrib[j]), f"T={T} pair {k}: an update of column {j} is not ordered before it"
                assert sum(c[2] - c[1] for c in contrib[j]) == k, f"T={T} pair {k}: column {j} has {contrib[j]} before its chain"
            if k + 1 < T:
                contrib[k + 1].append((i, k, k + 1, SIDE))
            for j in cols:
                done[j] = i
                writes[i] |= 1 << j
                reads[i] |= 1 << j
        elif op == POP_UPDATE:
            assert 1 <= nc <= MAX_COLS and j0 + nc <= T
            assert all(kb[c] >= kb[c + 1] for c in range(nc - 1)), f"T={T} op {i}: kb {kb} grows to the right (longest K first)"
            for c in range(nc):
                j = j0 + c
                assert 0 <= kb[c] < kend <= j, f"T={T} op {i}: column {j} panels [{kb[c]}, {kend})"
                for p in range(kb[c], kend):
                    assert p in done and (a >> done[p]) & 1, f"T={T} op {i}: reads panel {p} before its chain is ordered before it"
                contrib[j].append((i, kb[c], kend, st))
                writes[i] |= 1 << j
                reads[i] |= 1 << j
                # algorithmic flops: lower triangle incl. diagonal of block column j, 2 flops per MAC, K = 128 per panel
                if st == MAIN:
                    main_flops += 2.0 * (NB * (T - j) * NB - NB * (NB - 1) / 2) * NB * (kend - kb[c])
            reads[i] |= ((1 << kend) - 1) ^ ((1 << min(kb)) - 1)
        else:
            assert op == POP_WAIT
    # every block column j > 0 takes panels 0 .. j-1 exactly once, in ascending contiguous ranges, each range ordered
    # after the previous one; panels of j's own quad on the side stream, the rest on the main stream
    for j in range(1, T):
        pos = 0
        prev = None
        for (i, p0, p1, st) in contrib[j]:
            assert p0 == pos and p1 > p0, f"T={T} column {j}: ranges {[(c[1], c[2]) for c in contrib[j]]}"
            if prev is not None:
                assert (anc[i] >> prev) & 1, f"T={T} column {j}: op {i} not ordered after op {prev}"
            quad0 = 4 * (j // 4)
            assert (st == SIDE) == (p0 >= quad0) and (p1 <= quad0 or p0 >= quad0), f"T={T} column {j}: [{p0}, {p1}) on stream {st}"
            pos, prev = p1, i
        assert pos == j, f"T={T} column {j} ends at panel {pos}"
    assert sorted(done) == list(range(T))
    # operations that are not ordered touch disjoint block columns (writes against reads and writes)
    for i in range(n):
        for m in range(i):
            if (anc[i] >> m) & 1:
                continue
            assert not (writes[i] & (reads[m] | writes[m])) and not (writes[m] & reads[i]), \
                f"T={T}: ops {m} and {i} are unordered and share block columns"
    # the whole factorisation ends on the main stream
    assert ops[-1][0] == POP_WAIT and ops[-1][1] == MAIN
    assert (anc[n - 1] & ((1 << n) - 1)) == (1 << n) - 1
    return main_flops


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("T", list(range(1, 41)) + [128])
def test_potrf_plan(lib, T, sms):
    import bench
    flops = check_plan(plan(lib, T, sms), T)
    assert flops == pytest.approx(bench.syrk_flops_per_fit(NB * T), rel=1e-12, abs=0)


def test_potrf_plan_passes_hold_the_fill(lib):
    """At N = 16384 on 132 SMs every deferred pass either reaches eight waves of CTAs or runs to the last block column."""
    T, sms = 128, 132
    ops = plan(lib, T, sms)
    upd = [r for r in ops if r[0] == POP_UPDATE and r[1] == MAIN]
    ll = upd[1::2]
    assert len(ll) == (T + 3) // 4 - 2
    for r in ll:
        j0, nc = int(r[3]), int(r[4])
        ctas = 2 * sum(T - j for j in range(j0, j0 + nc))
        assert ctas >= 8 * 2 * sms or j0 + nc == T or nc == MAX_COLS
        assert nc >= min(4, T - j0)
