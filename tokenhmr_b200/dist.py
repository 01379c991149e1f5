"""Batch sharding over the GPUs of one box (SURVEY.md §8e).

Every image is independent from batch['img'] to every output (LayerNorm / softmax are per-row, no BatchNorm on
the path), so the data path needs no collective: rank r owns a contiguous slice of the batch and the weights
are replicated.  The one exchange step is an all-gather of the per-image outputs so that every rank sees the
whole batch (BASELINE.json configs[2]).  `cls_logits_softmax` (1.3 MB/image) is not gathered by default.

Two transports behind the same host logic (shard ranges, padding of uneven shards, trimming):

* native (TokenHMREngine on CUDA): the in-place design of SURVEY.md §8e.  Each gathered field is one device buffer of
  world * rows images; the engine writes this rank's images straight into its rows and `thmr_allgather_outputs`
  (C ABI, include/tokenhmr_b200.h) issues one grouped ncclAllGather with sendbuff = recvbuff + rank * count on the
  forward's stream, inside the same CUDA graph.  No pack / unpack copies, no torch collective.  The NCCL communicator
  is created by the library from a unique id that rank 0 broadcasts over torch.distributed.
* torch (any callable model, any backend incl. gloo on CPU): one packed, padded buffer per rank and
  torch.distributed.all_gather_into_tensor.  Used by the CPU tests of the host logic and by non-engine models.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from . import _lib

# (output key, per-image shape) in packing order; shapes are filled from the first output dict
GATHER_KEYS = ["pred_vertices", "pred_keypoints_3d", "pred_keypoints_2d", "pred_cam", "pred_cam_t", "focal_length",
               "global_orient", "body_pose", "betas"]


def shard_range(global_batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous split; the first (global_batch % world) ranks take one extra image."""
    base, rem = divmod(global_batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_sizes(global_batch: int, world: int) -> List[int]:
    return [hi - lo for lo, hi in (shard_range(global_batch, r, world) for r in range(world))]


def _flat_outputs(out: Dict) -> Dict[str, torch.Tensor]:
    flat = {k: v for k, v in out.items() if isinstance(v, torch.Tensor)}
    flat.update(out.get("pred_smpl_params", {}))
    return flat


def pack(out: Dict, rows: int, buf: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, List[Tuple[str, torch.Size, int]]]:
    """Struct-of-arrays packing of one rank's outputs into one contiguous fp32 buffer with `rows` image slots per
    field (rows >= local batch; the tail of each field is padding so that every rank sends the same count)."""
    flat = _flat_outputs(out)
    layout, total = [], 0
    for k in GATHER_KEYS:
        t = flat[k]
        per = t[0].numel()
        layout.append((k, t.shape[1:], per))
        total += per * rows
    if buf is None or buf.numel() != total:
        buf = torch.zeros(total, device=flat[GATHER_KEYS[0]].device, dtype=torch.float32)
    off = 0
    for k, _, per in layout:
        n = flat[k].shape[0]
        if n > rows:
            raise ValueError(f"local batch {n} exceeds the {rows} rows reserved per rank")
        buf[off:off + n * per].copy_(flat[k].reshape(-1))
        off += per * rows
    return buf, layout


def trim(parts: Dict[str, torch.Tensor], rows: int, sizes: Sequence[int]) -> Dict[str, torch.Tensor]:
    """parts[k]: (world * rows, ...) with rank r's images in rows [r*rows, r*rows + sizes[r]) -> (sum(sizes), ...).
    Equal full shards need no copy."""
    if all(n == rows for n in sizes):
        return parts
    dev = next(iter(parts.values())).device
    idx = torch.cat([torch.arange(r * rows, r * rows + n) for r, n in enumerate(sizes)]).to(dev)
    return {k: v.index_select(0, idx) for k, v in parts.items()}


def unpack(gathered: torch.Tensor, layout, rows: int, sizes: Sequence[int]) -> Dict[str, torch.Tensor]:
    """gathered: (world, total) -> dict of (sum(sizes), ...) tensors."""
    world = gathered.shape[0]
    parts, off = {}, 0
    for k, shape, per in layout:
        parts[k] = gathered[:, off:off + per * rows].reshape(world * rows, *shape)
        off += per * rows
    return _as_output_dict(trim(parts, rows, sizes))


def _as_output_dict(parts: Dict[str, torch.Tensor]) -> Dict:
    res = {k: v for k, v in parts.items() if k not in ("global_orient", "body_pose", "betas")}
    res["pred_smpl_params"] = {k: parts[k] for k in ("global_orient", "body_pose", "betas")}
    return res


class ShardedTokenHMR:
    """Runs the local shard through `model` and all-gathers the outputs (one collective per forward).

        sharded = ShardedTokenHMR(model)                 # after dist.init_process_group(...)
        lo, hi = shard_range(global_batch, rank, world)
        out = sharded({"img": img[lo:hi]})               # every rank gets the outputs of all `global_batch` images

    Shards may be uneven (global batch not divisible by the world size): every rank reserves rows = max shard and the
    padding rows are trimmed after the exchange.  The shard sizes are exchanged once per distinct local batch size."""

    def __init__(self, model, group=None, transport: str = "auto", gather_logits: bool = False):
        self.model = model
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        from .engine import TokenHMREngine
        native_ok = isinstance(model, TokenHMREngine)
        if transport == "auto":
            transport = "native" if native_ok else "torch"
        if transport == "native" and not native_ok:
            raise ValueError("the native transport needs a TokenHMREngine")
        self.transport = transport
        self.gather_logits = bool(gather_logits)
        if self.gather_logits and not getattr(model, "has_logits", True):
            raise _lib.ThmrError("gather_logits=True: a regression-head (transformer_decoder) model produces no "
                                 "cls_logits_softmax")
        self._comm = None
        self._sizes: Dict[int, List[int]] = {}
        self._send = None
        self._recv = None
        if transport == "native":
            self._init_comm()

    # ------------------------------------------------------------------------------------------ native transport
    def _init_comm(self) -> None:
        from ._lib import check, lib
        ident = [None]
        if self.rank == 0:
            buf = ctypes.create_string_buffer(128)
            check(lib().thmr_comm_unique_id(buf))
            ident = [buf.raw]
        if self.world > 1:
            dist.broadcast_object_list(ident, src=dist.get_global_rank(self.group, 0) if self.group is not None else 0,
                                       group=self.group)
        h = ctypes.c_void_p()
        with torch.cuda.device(self.model.device):
            check(lib().thmr_comm_create(ident[0], self.world, self.rank, ctypes.byref(h)))
        self._comm = h

    def close(self) -> None:
        """Destroy the library's communicator.  CUDA graphs that captured its collectives keep the communicator alive
        (ncclCommDestroy would wait for them forever), so the engine's sharded buffer sets -- and with them their graphs --
        are released first."""
        if self._comm:
            from ._lib import lib
            m = self.model
            for key in [k for k, st in m._bufs.items() if st.get("shard") is not None]:
                st = m._bufs.pop(key)
                st["graph"] = None
            torch.cuda.synchronize(m.device)
            comm, self._comm = self._comm, None
            lib().thmr_comm_destroy(comm)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def spec(self, local_batch: int):
        """ShardSpec for a local batch of this size (exchanges the shard sizes of all ranks the first time)."""
        from .engine import ShardSpec
        sizes = self.sizes(local_batch)
        return ShardSpec(self._comm.value, self.world, self.rank, max(sizes), self.gather_logits)

    # ------------------------------------------------------------------------------------------ shared host logic
    def sizes(self, local_batch: int) -> List[int]:
        s = self._sizes.get(local_batch)
        if s is None:
            if self.world == 1:
                s = [local_batch]
            else:
                got: List = [None] * self.world
                dist.all_gather_object(got, int(local_batch), group=self.group)
                s = [int(v) for v in got]
            self._sizes[local_batch] = s
        return s

    def forward_local(self, batch: Dict) -> Dict:
        return self.model(batch)

    def all_gather(self, out: Dict, sizes: Optional[Sequence[int]] = None) -> Dict:
        """torch transport: pack (padded to the largest shard) + one all_gather_into_tensor + trim."""
        n = _flat_outputs(out)[GATHER_KEYS[0]].shape[0]
        sizes = list(sizes) if sizes is not None else self.sizes(n)
        rows = max(sizes)
        self._send, layout = pack(out, rows, self._send)
        if self.world == 1:
            return unpack(self._send.unsqueeze(0), layout, rows, sizes)
        if self._recv is None or self._recv.numel() != self.world * self._send.numel():
            self._recv = torch.empty(self.world, self._send.numel(), device=self._send.device, dtype=torch.float32)
        dist.all_gather_into_tensor(self._recv.view(-1), self._send, group=self.group)
        return unpack(self._recv, layout, rows, sizes)

    def __call__(self, batch: Dict, **kw) -> Dict:
        """batch['img'] is this rank's shard; returns the gathered outputs of the whole global batch."""
        if self.transport == "torch":
            return self.all_gather(self.forward_local(batch))
        n = batch["img"].shape[0]
        spec = self.spec(n)
        out = self.model.forward(batch, shard=spec, **kw)
        sizes = self.sizes(n)
        parts = {k: out[k] for k in GATHER_KEYS if k in out}
        parts.update(out["pred_smpl_params"])
        res = _as_output_dict(trim(parts, spec.rows, sizes))
        if self.gather_logits:
            res["cls_logits_softmax"] = trim({"p": out["cls_logits_softmax"]}, spec.rows, sizes)["p"]
        elif "cls_logits_softmax" in out:
            res["cls_logits_softmax_local"] = out["cls_logits_softmax"]
        return res
