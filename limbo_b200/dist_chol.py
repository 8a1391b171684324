"""Multi-GPU Cholesky of the GP kernel matrix (BASELINE.json config 5: N = 65536 on 8 GPUs; SURVEY.md §8e).

The factor `Eigen::LLT<MatrixXd>(_kernel).matrixL()` (model/gp.hpp:565) of one GP is distributed 1-D block-cyclically
over 256-column panels ("pairs" of 128-blocks): pair p lives on rank p mod G, full height, so K never exists in one
place — every rank generates its own columns from X.  One step of the right-looking factorisation:

    owner          : factor the pair (potf2 / trsm / K=128 column update / potf2 / trsm on the fp64 tensor cores),
                     pack the rows below it into a contiguous panel                       [lb_dchol_panel, side stream]
    all ranks      : broadcast of the panel — the ONE exchange step of the path            [NCCL, communication stream]
    all ranks      : K = 256 trailing update of the local columns right of the pair         [lb_dchol_update, main stream]

with look-ahead: the owner of pair p+1 updates that pair first ("a" part), factors and ships it while everybody is
still in the "b" part of update p.  Panels are double buffered.  `schedule()` is the rank-independent action list
(tested on CPU with gloo and a NumPy executor in tests/test_dist_gloo.py); `DistCholesky` executes it with CUDA streams
and torch.distributed (NCCL) — there is no CPU path in the product.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

TILE = 128
PAIR = 2 * TILE


_PANEL_GROUP = None


def panel_group():
    """Process group for the panel broadcasts whose NCCL kernels run on a HIGH-PRIORITY stream.  The trailing update keeps
    every SM full (two resident CTAs per SM, thousands of blocks pending); a broadcast kernel launched at default priority is
    only scheduled once the update has drained, i.e. the exchange step would not overlap the update at all.  Collective: every rank must
    call it (DistCholesky does, at construction).  Falls back to the default group when the option is unavailable."""
    global _PANEL_GROUP
    import torch.distributed as dist
    if _PANEL_GROUP is None:
        try:
            opts = dist.ProcessGroupNCCL.Options(is_high_priority_stream=True)
            _PANEL_GROUP = dist.new_group(backend="nccl", pg_options=opts)
        except Exception:
            _PANEL_GROUP = dist.group.WORLD
    return _PANEL_GROUP


def padded_order(n: int) -> int:
    return (n + PAIR - 1) // PAIR * PAIR


def local_pairs(npairs: int, rank: int, world: int) -> list[int]:
    return list(range(rank, npairs, world))


def global_block(l: int, rank: int, world: int) -> int:
    """global 128-block column of local block column l (potrf.cu: dchol_global_block)"""
    return 2 * (world * (l // 2) + rank) + (l & 1)


def schedule(npairs: int, rank: int, world: int):
    """Yields the actions of `rank`, in issue order:
        ("panel", p)                 factor pair p (owner only) and pack its panel into buffer p % 2
        ("bcast", p, owner)          broadcast panel p (buffer p % 2) from owner
        ("update", p, l0, l1, tag)   update local block columns [l0, l1) with panel p; tag "a" = look-ahead columns of
                                     the next pair (the next panel waits for it), "b" = the rest
    The last pair has nothing below it: no broadcast, no update."""
    mine = local_pairs(npairs, rank, world)
    nlb = 2 * len(mine)
    for p in range(npairs):
        owner = p % world
        if owner == rank:
            yield ("panel", p)
        if p == npairs - 1:
            break
        yield ("bcast", p, owner)
        nxt = p + 1
        if nxt % world == rank:
            la = 2 * (nxt // world)
            yield ("update", p, la, la + 2, "a")
            if la + 2 < nlb:
                yield ("update", p, la + 2, nlb, "b")
        else:
            # first local pair right of p
            lp = next((i for i, q in enumerate(mine) if q > p), None)
            if lp is not None:
                yield ("update", p, 2 * lp, nlb, "b")


class DistCholesky:
    """Distributed factor of K(X, X) + (noise + 1e-8) I for the kernel functor `kernel_fn` (limbo_b200.kernel.*).
    One instance per rank (torchrun); `factor()` leaves this rank's columns of L in `self.L` (shape (ncols_local, Nd),
    i.e. the column-major Nd x ncols_local block) with a zero upper triangle, and returns (info, log det K)."""

    def __init__(self, X: np.ndarray, kernel_fn, rank: int, world: int, device, group=None):
        import torch
        from . import _lib
        self._torch = torch
        if group is None and world > 1:
            import torch.distributed as dist
            if dist.is_initialized() and dist.get_backend() == "nccl":
                group = panel_group()
        self.rank, self.world, self.group = rank, world, group
        self.device = torch.device(device)
        self.N, self.D = X.shape
        self.Nd = padded_order(self.N)
        self.T = self.Nd // TILE
        self.npairs = self.T // 2
        self.pairs = local_pairs(self.npairs, rank, world)
        self.ncols = PAIR * len(self.pairs)
        lib = _lib.load()
        self._lib = lib
        vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
        lib.lb_dchol_set_points.argtypes = [vp, i64, i32, vp]
        lib.lb_dchol_build.argtypes = [vp, i64, i32, i32, i64, vp]
        lib.lb_dchol_panel.argtypes = [vp, vp, i64, i32, vp, vp, vp]
        lib.lb_dchol_update.argtypes = [vp, vp, i64, vp, i32, i32, i32, i32, i32]
        lib.lb_dchol_finish.argtypes = [vp, vp, i64, i64, i32, i32, i64, vp]
        for f in ("lb_dchol_set_points", "lb_dchol_build", "lb_dchol_panel", "lb_dchol_update", "lb_dchol_finish"):
            getattr(lib, f).restype = i32
        dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.main = torch.cuda.Stream(self.device)
        self.side = torch.cuda.Stream(self.device, priority=-1)
        self.comm = torch.cuda.Stream(self.device, priority=-1)
        self._h_main, self._h_side = vp(), vp()
        _lib.check(lib.lb_create(C.byref(self._h_main), dev_index, 0), "lb_create")
        _lib.check(lib.lb_create(C.byref(self._h_side), dev_index, 0), "lb_create")
        _lib.check(lib.lb_set_stream(self._h_main, self.main.cuda_stream), "lb_set_stream")
        _lib.check(lib.lb_set_stream(self._h_side, self.side.cuda_stream), "lb_set_stream")
        Xc = np.ascontiguousarray(X, dtype=np.float64)
        _lib.check(lib.lb_dchol_set_points(self._h_main, self.N, self.D, Xc.ctypes.data), "lb_dchol_set_points")
        own = np.ascontiguousarray(kernel_fn.params(), dtype=np.float64)
        _lib.check(lib.lb_set_kernel(self._h_main, kernel_fn.kernel_id, own.ctypes.data, own.size, kernel_fn.noise()), "lb_set_kernel")
        f64 = torch.float64
        self.L = torch.empty((max(self.ncols, 1), self.Nd), dtype=f64, device=self.device)
        self.panels = [torch.empty(PAIR * max(self.Nd - PAIR, 1), dtype=f64, device=self.device) for _ in range(2)]
        self.invD = torch.zeros(2 * TILE * TILE, dtype=f64, device=self.device)
        self.info = torch.zeros(2, dtype=torch.int32, device=self.device)
        self.logdet_part = torch.zeros(1, dtype=f64, device=self.device)
        self.launches = 0

    def close(self) -> None:
        for h in (self._h_main, self._h_side):
            if h is not None and h.value:
                self._lib.lb_destroy(h)
        self._h_main = self._h_side = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- pieces ---------------------------------------------------------------------------------------------
    def build(self) -> None:
        """Generate this rank's columns of K (kernel.hpp:81-84 incl. noise + 1e-8 on the diagonal)."""
        from . import _lib
        if self.ncols:
            _lib.check(self._lib.lb_dchol_build(self._h_main, self.Nd, self.rank, self.world, self.ncols, self.L.data_ptr()), "lb_dchol_build")

    def _ldp(self, p: int) -> int:
        return self.Nd - (2 * p + 2) * TILE

    def factor(self):
        """Runs the schedule.  Returns (info, logdet): info = 0 or the 1-based index of the first non-positive pivot
        (LAPACK style, like lb_fit); logdet = 2 sum log L_jj over all ranks (one all_reduce)."""
        import torch.distributed as dist
        from . import _lib
        torch = self._torch
        lib = self._lib
        Ev = torch.cuda.Event
        ev_a = Ev()          # the pair about to be factored has received all its updates
        ev_panel = Ev()      # panel packed (owner)
        ev_bcast = Ev()      # panel arrived
        ev_free = [None, None]  # buffer last read by an update
        # optional per-step timeline (LB_DCHOL_TIMELINE=<file prefix>): CUDA timing events at the end of every panel,
        # broadcast and update of this rank, dumped as JSON after the run (diagnosis of the critical path; not used by the product)
        import os as _os
        tl_prefix = _os.environ.get("LB_DCHOL_TIMELINE")
        tl = [] if tl_prefix else None

        def mark(tag, p, stream):
            if tl is not None:
                e = Ev(enable_timing=True)
                e.record(stream)
                tl.append((tag, p, e))
        with torch.cuda.stream(self.main):
            self.info.zero_()  # on the stream whose kernels consume it (not torch's current stream)
        self.side.wait_stream(self.main)
        ev_a.record(self.main)  # after build()
        mark("start", -1, self.main)
        have_a = True
        for act in schedule(self.npairs, self.rank, self.world):
            kind, p = act[0], act[1]
            buf = self.panels[p % 2]
            if kind == "panel":
                lp = p // self.world
                cols = self.L.data_ptr() + 8 * lp * PAIR * self.Nd
                if have_a:
                    self.side.wait_event(ev_a)
                if ev_free[p % 2] is not None:
                    self.side.wait_event(ev_free[p % 2])  # the pack overwrites the buffer update p-2 read
                _lib.check(lib.lb_dchol_panel(self._h_side, cols, self.Nd, 2 * p, self.invD.data_ptr(), self.info.data_ptr(),
                                              buf.data_ptr()), "lb_dchol_panel")
                ev_panel.record(self.side)
                mark("panel", p, self.side)
            elif kind == "bcast":
                owner = act[2]
                n = PAIR * self._ldp(p)
                with torch.cuda.stream(self.comm):
                    if owner == self.rank:
                        self.comm.wait_event(ev_panel)
                    elif ev_free[p % 2] is not None:
                        self.comm.wait_event(ev_free[p % 2])
                    if self.world > 1:
                        dist.broadcast(buf[:n], src=owner, group=self.group)
                    ev_bcast.record(self.comm)
                    mark("bcast", p, self.comm)
                self.main.wait_event(ev_bcast)
            else:
                _, _, l0, l1, tag = act
                _lib.check(lib.lb_dchol_update(self._h_main, self.L.data_ptr(), self.Nd, buf.data_ptr(), 2 * p, l0, l1, self.rank,
                                               self.world), "lb_dchol_update")
                if tag == "a":
                    ev_a.record(self.main)
                mark("update_" + tag, p, self.main)
                e = Ev()
                e.record(self.main)
                ev_free[p % 2] = e
        self.main.wait_stream(self.side)
        self.main.wait_stream(self.comm)
        _lib.check(lib.lb_dchol_finish(self._h_main, self.L.data_ptr(), self.Nd, self.N, self.rank, self.world, self.ncols,
                                       self.logdet_part.data_ptr()), "lb_dchol_finish")
        with torch.cuda.stream(self.main):
            rec = torch.stack([self.logdet_part[0], self.info[0].to(torch.float64)])
            if self.world > 1:
                # the ONE small reduction: [sum, max] packed as two all_reduces would be two collectives; gather instead
                out = [torch.zeros_like(rec) for _ in range(self.world)]
                dist.all_gather(out, rec, group=self.group)
                allrec = torch.stack(out)
            else:
                allrec = rec[None]
        self.main.synchronize()
        allrec = allrec.cpu().numpy()
        infos = allrec[:, 1][allrec[:, 1] > 0]
        self.launches = int(lib.lb_launch_count(self._h_main) + lib.lb_launch_count(self._h_side))
        if tl is not None:
            import json as _json
            torch.cuda.synchronize(self.device)
            t0 = tl[0][2]
            rows = [[tag, p, t0.elapsed_time(e)] for tag, p, e in tl]
            with open(f"{tl_prefix}_rank{self.rank}.json", "w") as f:
                _json.dump({"world": self.world, "N": self.N, "events_ms": rows}, f)
        return (int(infos.min()) if infos.size else 0), float(2.0 * allrec[:, 0].sum())

    # ---- helpers for checks ----------------------------------------------------------------------------------
    def global_columns(self) -> np.ndarray:
        """global column index of every local column"""
        cols = []
        for l in range(2 * len(self.pairs)):
            j = global_block(l, self.rank, self.world)
            cols.extend(range(j * TILE, (j + 1) * TILE))
        return np.asarray(cols, dtype=np.int64)
