"""Inversion of the factor spread over the ranks, for the reduced-precision candidate path (BASELINE.json config 4 on several
GPUs).  sigma^2(v) = k(v,v) - |L^-1 k(v)|^2 (model/gp.hpp:618-624) is scored on the wgmma path against a reduced-precision copy
of ALL of L^-1 on every rank, the candidates being sharded (limbo_b200.dist.sharded_acq_argmax).  Inverting the whole factor on
every rank would be the Amdahl term once the fit is distributed (dist_fit.py).  The columns of a triangular inverse
are independent, so here rank r computes the 128-column tiles r, r + G, r + 2G, ... with the blocked solve of the batched query
path on identity columns (N^3 / (3 G) flops on the fp64 tensor cores), casts them to the storage type of the handle's precision,
and ONE all_gather of the chunks (N^2 / G reduced-precision elements per rank) gives every rank the whole copy.

    prepare(gp)   =  lb_dinv_columns  ->  all_reduce(max |.|)  [fp16 scale]  ->  lb_dinv_pack  ->  all_gather  ->  lb_dinv_adopt

There is no CPU path; world == 1 runs the same kernels on one GPU (single-GPU tests: tests/test_gpu_dist_inv.py, which also
drives G = 2, 3 chunk by chunk on one device)."""
from __future__ import annotations

import ctypes as C

from . import _lib


TILE = 128


def owned_tiles(T: int, rank: int, world: int) -> list[int]:
    """global 128-column tiles of L^-1 computed by `rank` (tile-cyclic: local tile t is global tile rank + t * world)"""
    return list(range(rank, T, world))


def chunk_layout(Np: int, world: int, precision: str) -> dict:
    """Byte layout of one rank's chunk (what the all_gather moves; include/limbo_b200_dist.h, lb_dinv_pack):
    [ hi plane: Np x W row-major | lo plane (fp16x3 only) | W float64 column weights |L^-1 e_k|^2 ],  W = 128 * ceil(T / world)."""
    T = Np // TILE
    W = TILE * ((T + world - 1) // world)
    elem = 4 if precision == "tf32" else 2          # tf32 values travel as fp32 words
    planes = 2 if precision == "fp16x3" else 1
    plane_bytes = Np * W * elem
    return {"width": W, "elem_bytes": elem, "planes": planes, "plane_bytes": plane_bytes, "weights_offset": planes * plane_bytes,
            "chunk_bytes": planes * plane_bytes + 8 * W}


def bind(lib):
    vp, i32, f64 = C.c_void_p, C.c_int, C.c_double
    lib.lb_dinv_chunk_bytes.argtypes = [vp, i32]
    lib.lb_dinv_chunk_bytes.restype = C.c_longlong
    lib.lb_dinv_columns.argtypes = [vp, i32, i32, C.POINTER(f64)]
    lib.lb_dinv_pack.argtypes = [vp, i32, i32, f64, vp]
    lib.lb_dinv_adopt.argtypes = [vp, i32, vp, f64]
    for f in ("lb_dinv_columns", "lb_dinv_pack", "lb_dinv_adopt"):
        getattr(lib, f).restype = i32
    return lib


class DistInverse:
    """prepare(gp): all ranks call it after the fit (lb_fit or DistFit.fit) of a reduced-precision limbo_b200.model.GP with the
    same samples and hyper-parameters; the next query_batch / argmax_batch on gp then scores without inverting anything."""

    def __init__(self, gp, rank: int, world: int, device, group=None):
        import torch
        self.rank, self.world, self.group = int(rank), int(world), group
        self.device = torch.device(device)
        self._lib = bind(_lib.load())
        self._torch = torch
        self._chunk = None
        self._all = None
        self._mx = torch.zeros(1, dtype=torch.float64, device=self.device)

    def supported(self, gp) -> bool:
        return gp._precision in (1, 2, 3) and gp.nb_samples() > 0  # tf32 / fp16 / fp16x3 handles

    def _buffers(self, nbytes: int):
        torch = self._torch
        if self._chunk is None or self._chunk.numel() != nbytes:
            self._all = torch.empty(self.world * nbytes, dtype=torch.uint8, device=self.device)
            self._chunk = torch.empty(nbytes, dtype=torch.uint8, device=self.device) if self.world > 1 else self._all
        return self._chunk, self._all

    def prepare(self, gp) -> None:
        torch, lib, h = self._torch, self._lib, gp._h
        import torch.distributed as dist
        nbytes = int(lib.lb_dinv_chunk_bytes(h, self.world))
        if nbytes <= 0:
            _lib.check(int(nbytes), "lb_dinv_chunk_bytes")
        chunk, everything = self._buffers(nbytes)
        mx = C.c_double(0.0)
        _lib.check(lib.lb_dinv_columns(h, self.rank, self.world, C.byref(mx)), "lb_dinv_columns")  # synchronises the handle's stream
        amax = float(mx.value)
        multi = self.world > 1 and dist.is_available() and dist.is_initialized()
        if multi:
            self._mx.fill_(amax)
            dist.all_reduce(self._mx, op=dist.ReduceOp.MAX, group=self.group)
            amax = float(self._mx.item())
        _lib.check(lib.lb_dinv_pack(h, self.rank, self.world, amax, chunk.data_ptr()), "lb_dinv_pack")
        if multi:
            _lib.check(lib.lb_sync(h), "lb_sync")  # the pack runs on the handle's stream, the collective on torch's
            dist.all_gather_into_tensor(everything, chunk, group=self.group)
            torch.cuda.current_stream(self.device).synchronize()
        _lib.check(lib.lb_dinv_adopt(h, self.world, everything.data_ptr(), amax), "lb_dinv_adopt")

    def close(self) -> None:
        self._chunk = self._all = None
