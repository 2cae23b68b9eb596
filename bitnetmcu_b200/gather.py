"""Result exchange of the sharded batch (SURVEY.md 8e), device tensors end to end.

The path itself has no collective: rank r infers its contiguous slice and the int32 class scores stay in its HBM.  A caller
that needs the results in one place has three ways to get them, all measured by ``bench.py --gpus N`` (`gather` object):

* ``nccl``      -- ``all_gather_into_tensor`` of the labels / logits after the kernel (serial: the baseline);
* ``p2p``       -- the fused kernel's epilogue stores each label (and optionally each logits row) straight into the gather
                  buffers of the peers through NVLink (CUDA IPC-mapped peer memory, ``bnm_infer_batch_device_gather``): the
                  exchange rides under the compute, no second kernel, no NCCL on the data path;
* ``none``      -- results stay sharded.

An all-gathered logits tensor is NVLink-ingest bound whatever the kernels do: every GPU receives 40 B per image of the other
ranks, so the box tops out at the NVLink ingest bandwidth / 40 B images/s per destination; labels (4 B/image) scale.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import numpy as np

from . import _lib
from .engine import N


class _DevArray:
    """Device memory owned by the C ABI (cudaMalloc: exportable through CUDA IPC), viewable as a torch tensor without a copy."""

    def __init__(self, ptr: int, shape, typestr: str, owner=None):
        self.ptr, self.shape, self.typestr, self._owner = ptr, tuple(shape), typestr, owner
        self.__cuda_array_interface__ = {"shape": self.shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


class PeerGatherBuffers:
    """Per-rank gather buffers (labels uint32 [world * n], optionally logits int32 [world * n][C]) that every peer maps.

    rank r's kernel writes rows [r * n, (r + 1) * n) of EVERY destination's buffers (all-gather semantics) or of the root's
    only.  Construction is collective (handles are exchanged with ``all_gather_object``)."""

    def __init__(self, n_per_rank: int, n_classes: int, device: int, with_logits: bool = True, group=None):
        import torch
        import torch.distributed as dist
        self.lib = _lib.load()
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.n, self.C, self.device = n_per_rank, n_classes, device
        rows = self.world * n_per_rank
        self._local_ptrs = []

        def alloc(nbytes):
            p = C.c_void_p()
            _lib.check(self.lib.bnm_device_alloc(device, nbytes, C.byref(p)), "bnm_device_alloc")
            self._local_ptrs.append(p.value)
            return p.value
        self.lab_ptr = alloc(rows * 4)
        self.lab8_ptr = alloc(rows)                  # one byte per label (n_classes <= 255): a quarter of the NVLink traffic
        self.log_ptr = alloc(rows * n_classes * 4) if with_logits else None

        def export(ptr):
            h = (C.c_ubyte * 64)()
            _lib.check(self.lib.bnm_ipc_export(C.c_void_p(ptr), h), "bnm_ipc_export")
            return bytes(h)
        mine = {"lab": export(self.lab_ptr), "lab8": export(self.lab8_ptr), "log": export(self.log_ptr) if with_logits else None}
        allh: List[Optional[dict]] = [None] * self.world
        dist.all_gather_object(allh, mine, group=group)
        self._opened = []
        self.lab_dst: List[int] = []
        self.lab8_dst: List[int] = []
        self.log_dst: List[int] = []
        for r, h in enumerate(allh):
            if r == self.rank:
                self.lab_dst.append(self.lab_ptr)
                self.lab8_dst.append(self.lab8_ptr)
                self.log_dst.append(self.log_ptr or 0)
                continue
            p = C.c_void_p()
            _lib.check(self.lib.bnm_ipc_open(device, (C.c_ubyte * 64).from_buffer_copy(h["lab"]), C.byref(p)), "bnm_ipc_open")
            self._opened.append(p.value)
            self.lab_dst.append(p.value)
            p8 = C.c_void_p()
            _lib.check(self.lib.bnm_ipc_open(device, (C.c_ubyte * 64).from_buffer_copy(h["lab8"]), C.byref(p8)), "bnm_ipc_open")
            self._opened.append(p8.value)
            self.lab8_dst.append(p8.value)
            if with_logits:
                q = C.c_void_p()
                _lib.check(self.lib.bnm_ipc_open(device, (C.c_ubyte * 64).from_buffer_copy(h["log"]), C.byref(q)), "bnm_ipc_open")
                self._opened.append(q.value)
                self.log_dst.append(q.value)
            else:
                self.log_dst.append(0)
        dev = torch.device("cuda", device)
        self.labels = torch.as_tensor(_DevArray(self.lab_ptr, (rows,), "<i4", self), device=dev)
        self.labels_u8 = torch.as_tensor(_DevArray(self.lab8_ptr, (rows,), "|u1", self), device=dev)
        self.logits = torch.as_tensor(_DevArray(self.log_ptr, (rows, n_classes), "<i4", self), device=dev) if with_logits else None

    def spec(self, labels_to: Optional[List[int]], logits_to: Optional[List[int]], labels_u8: bool = False):
        """bnm_gather for this rank: destination ranks of the labels / logits (None = nobody); labels_u8: one byte per label."""
        g = _lib.BnmGather()
        g.row_offset = self.rank * self.n
        g.labels_u8 = 1 if labels_u8 else 0
        for k, r in enumerate(labels_to or []):
            g.labels_dst[k] = (self.lab8_dst if labels_u8 else self.lab_dst)[r]
        g.n_labels_dst = len(labels_to or [])
        for k, r in enumerate(logits_to or []):
            g.logits_dst[k] = self.log_dst[r]
        g.n_logits_dst = len(logits_to or [])
        return g

    def close(self):
        for p in self._opened:
            self.lib.bnm_ipc_close(C.c_void_p(p))
        self._opened = []
        for p in self._local_ptrs:
            self.lib.bnm_device_free(C.c_void_p(p))
        self._local_ptrs = []


def infer_gather(eng, images, logits, labels, buffers: PeerGatherBuffers, labels_to, logits_to, stream: int, labels_u8: bool = False) -> None:
    """``Engine.infer_device`` whose epilogue also stores this rank's rows into the gather buffers of the ranks listed in
    ``labels_to`` / ``logits_to`` (pass this rank's own slice of its buffer as ``logits`` / ``labels`` and leave it out of the lists).
    ``logits`` / ``labels`` may be None: no local copy of that output (the call still needs one output or destination)."""
    import torch
    g = buffers.spec(labels_to, logits_to, labels_u8)
    eng._device_call(eng.lib.bnm_infer_batch_device_gather, images, torch.int8,
                     [(logits, torch.int32, (N, eng.n_classes)), (labels, 4, N), C.byref(g)], stream)


def bench_gathers(ctx, eng, db, ms_compute: float) -> dict:
    """Timings of the result exchange at N > 1 for bench.py: serial NCCL all-gathers (baseline) and the peer-store epilogue."""
    torch, tdist = ctx.torch, ctx.tdist
    n, C_, world, rank = db.n, eng.n_classes, ctx.world, ctx.rank
    out = {"backend": "nccl + CUDA IPC peer stores", "compute_ms_per_step_sharded": ms_compute}

    def timed(fn, reps=8, warm=2):
        for i in range(warm):
            fn(i)
        ctx.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(ctx.stream)
        for i in range(reps):
            fn(i)
        b.record(ctx.stream)
        ctx.barrier()
        return ctx.max_over_ranks(a.elapsed_time(b) / reps)

    # ---- baseline: NCCL all-gather after the kernel
    all_lab = torch.empty(n * world, dtype=torch.int32, device=ctx.dev)
    all_log = torch.empty((n * world, C_), dtype=torch.int32, device=ctx.dev)
    lab_ms = timed(lambda i: tdist.all_gather_into_tensor(all_lab, db.d_labels[0]))
    log_ms = timed(lambda i: tdist.all_gather_into_tensor(all_log, db.d_logits[0]))
    out["nccl_all_gather_labels_ms"] = lab_ms
    out["nccl_all_gather_logits_ms"] = log_ms
    out["value_with_label_gather_nccl_serial"] = world * n / ((ms_compute + lab_ms) * 1e-3)
    out["value_with_logits_gather_nccl_serial"] = world * n / ((ms_compute + log_ms) * 1e-3)
    del all_lab, all_log

    # ---- peer-store epilogue: this rank's rows go to its own slice of its gather buffer (the kernel's ordinary outputs) and, in the
    # same epilogue, to the same rows of the peers' buffers over NVLink.  labels to every rank (all-gather); logits to every rank /
    # to rank 0 only
    try:
        bufs = PeerGatherBuffers(n, C_, ctx.local_rank, with_logits=True)
        peers = [r for r in range(world) if r != rank]
        st = ctx.stream.cuda_stream
        my_log = bufs.logits[rank * n:(rank + 1) * n]
        my_lab = bufs.labels[rank * n:(rank + 1) * n]

        def run(labels_to, logits_to, u8=False):
            return timed(lambda i: infer_gather(eng, db.d_in[i & 1], my_log, my_lab, bufs, labels_to, logits_to, st, labels_u8=u8))

        def check(t_all, mine):   # after the barrier inside timed(): every rank's slice of MY buffer equals that rank's own slice
            theirs = [torch.empty_like(mine) for _ in range(world)]
            tdist.all_gather(theirs, mine.contiguous())
            return all(bool(torch.equal(t_all[r * n:(r + 1) * n], theirs[r])) for r in range(world))
        ms_lab = run(peers, None)
        out["value_with_label_gather"] = world * n / (ms_lab * 1e-3)
        out["label_gather_ms_per_step"] = ms_lab
        out["label_gather_complete_and_correct"] = check(bufs.labels, my_lab)
        ms_lab8 = run(list(range(world)), None, u8=True)   # one byte per label, every rank incl. this one (its own uint32 labels stay local)
        out["value_with_label_gather_u8"] = world * n / (ms_lab8 * 1e-3)
        out["label_gather_u8_ms_per_step"] = ms_lab8
        out["label_gather_u8_complete_and_correct"] = check(bufs.labels_u8, my_lab.to(torch.uint8))
        ms_log_all = run(peers, peers)
        out["value_with_logits_gather"] = world * n / (ms_log_all * 1e-3)
        out["logits_gather_ms_per_step"] = ms_log_all
        out["logits_gather_complete_and_correct"] = check(bufs.logits, my_log) and check(bufs.labels, my_lab)
        ms_log_root = run(None, [0] if rank != 0 else [])
        out["value_with_logits_gather_to_rank0"] = world * n / (ms_log_root * 1e-3)
        out["note"] = ("value_with_*_gather: every step's epilogue stores the rows into the peers' buffers over NVLink (labels: all ranks; logits: "
                       "all ranks, or rank 0 only); time = device events around the steps, max over ranks; the last step's images are the "
                       "same on every step parity, results compared rank by rank after a barrier; the headline value leaves results sharded")
        ctx.barrier()
        del my_log, my_lab
        bufs.close()
    except Exception as ex:
        out["p2p_error"] = str(ex)[:300]
    return out
