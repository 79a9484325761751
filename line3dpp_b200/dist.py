"""Multi-GPU matchImages: the exchange step behind L3DPP::Line3D::setShard (include/line3d.h, SURVEY.md §8(e)).

Every rank holds all images, matches its contiguous, cost-balanced share of the reference's view-pair list
(computeMatches order, line3D.cc:704-741) with `l3d_match_pairs_range`, and then needs the rows of the other ranks before
the order-dependent scoring sweep (storeInverseMatches, line3D.cc:1672-1699) can run replicated.  The rows live in two
device arrays with the layout of the FULL job (counts int32[rows], recs 24·knn B per row), so the exchange is one
broadcast per owner over NCCL/NVLink, in place, no packing.  Nothing else is communicated.  Keep-all (kNN <= 0) and
kNN > 32 exchange twice: the counts alone, which give every rank the same row stride, then the rows at that stride.
"""
from __future__ import annotations

import ctypes as C
import time

import numpy as np
import torch
import torch.distributed as dist

from . import capi

REC_BYTES = 24  # sizeof(l3d_match_rec)


class _DevArray:
    """a borrowed device allocation exposed through __cuda_array_interface__ so torch can wrap it without copying"""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3,
                                         "strides": None}


def device_bytes(ptr: int, nbytes: int, device: int) -> torch.Tensor:
    """uint8 view of `nbytes` of device memory at `ptr` (owned by the l3d context, which must outlive the tensor)"""
    if nbytes == 0:
        return torch.empty(0, dtype=torch.uint8, device=f"cuda:{device}")
    return torch.as_tensor(_DevArray(ptr, nbytes), device=f"cuda:{device}")


def balanced_split(cost, parts: int) -> np.ndarray:
    """bounds[parts+1] of the contiguous near-equal-cost split every rank computes identically (l3d_balanced_split)"""
    cost = np.ascontiguousarray(cost, np.int64)
    out = np.zeros(parts + 1, np.int32)
    rc = capi.lib().l3d_balanced_split(cost.ctypes.data_as(C.c_void_p), len(cost), int(parts), out.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise capi.L3DError(f"l3d_balanced_split failed ({rc})")
    return out


def exchange_rows(counts: torch.Tensor, recs: torch.Tensor, row_bounds, knn: int, group=None) -> None:
    """counts: uint8 view of int32[rows]; recs: uint8 view of rows*knn records.  Rank r owns rows
    [row_bounds[r], row_bounds[r+1]); after the call every rank holds every row.  knn = 0 (the first of the two calls of
    keep-all and kNN > 32, include/line3d.h) moves only the counts.  Works on CPU tensors (gloo) as well."""
    world = dist.get_world_size(group)
    assert len(row_bounds) == world + 1
    for r in range(world):
        a, b = int(row_bounds[r]), int(row_bounds[r + 1])
        if b <= a:
            continue
        src = dist.get_global_rank(group, r) if group is not None else r
        dist.broadcast(counts[4 * a:4 * b], src=src, group=group)
        if knn > 0:
            dist.broadcast(recs[REC_BYTES * knn * a:REC_BYTES * knn * b], src=src, group=group)


_EXCHANGE_T = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong), C.c_int, C.c_int)


def attach(line3d, device: int, group=None):
    """Make `line3d` (line3dpp_b200.line3d.Line3D) a member of the process group: matching sharded, the rest replicated.
    Returns the callback object, which the caller must keep alive as long as the Line3D is used.
    line3d._exchange_state["exchanges"] gets one entry per callback (knn, ms, count_bytes, record_bytes: what every rank holds
    after it); the caller may clear the list."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    state = {"error": None, "exchanges": []}

    def _exchange(_user, counts_dev, recs_dev, row_bounds, w, knn):
        try:
            rb = [row_bounds[i] for i in range(w + 1)]
            rows = rb[-1]
            counts = device_bytes(counts_dev, 4 * rows, device)
            recs = device_bytes(recs_dev, REC_BYTES * knn * rows, device)
            torch.cuda.synchronize(device)                     # the match kernel ran on the context's own stream
            t0 = time.perf_counter()
            exchange_rows(counts, recs, rb, knn, group)
            torch.cuda.synchronize(device)
            ms = (time.perf_counter() - t0) * 1e3              # the first call includes waiting for the slowest rank's matching
            state["exchange_ms"] = ms
            state["exchanges"].append({"knn": knn, "ms": ms, "count_bytes": 4 * rows, "record_bytes": REC_BYTES * knn * rows})
            return 0
        except Exception as e:  # noqa: BLE001 — must not unwind through the C frame
            state["error"] = e
            return -1

    cb = _EXCHANGE_T(_exchange)
    line3d._chk(line3d.L.l3dpp_set_shard(line3d.h, int(rank), int(world), cb, None), "setShard")
    line3d._exchange_cb, line3d._exchange_state = cb, state
    return cb
