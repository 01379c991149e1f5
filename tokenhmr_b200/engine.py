"""TokenHMREngine — drop-in for the reference's TokenHMR.forward(batch) -> dict surface.

Reference boundary (SURVEY.md §8b): tokenhmr/lib/models/tokenhmr.py:330-338 (forward) -> :135-188
(forward_step), built by load_tokenhmr (tokenhmr/lib/models/__init__.py:3-26) and called as
`model(batch)` under torch.no_grad() by demo.py:77-78, eval.py:146-147 and track.py:39.

    model = TokenHMREngine(cfg, state_dict, smpl_buffers, device='cuda:0')
    out = model({'img': img})          # img (B,3,256,256) fp32, any device; extra keys ignored
    out['pred_vertices'], out['pred_keypoints_3d'], out['pred_cam'], out['pred_smpl_params'], ...

Python here is host glue only (tensor allocation, dict packing, H2D of the input): every operation between
batch['img'] and the output tensors runs in libtokenhmr_b200.so through the C ABI, and fails loudly
if the library is missing.
"""
from __future__ import annotations

import ctypes
from typing import Dict, NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib
from ._lib import check, lib
from .config import TokenHMRConfig
from .ops import SMPLModel
from .weights import PackedWeights, make_config_struct


class ShardSpec(NamedTuple):
    """How this rank's forward sits in a batch sharded over `world` GPUs (tokenhmr_b200.dist.ShardedTokenHMR):
    every gathered output is one buffer of world * rows images, this rank writes rows [rank*rows, rank*rows + B)."""
    comm: int            # thmr_comm* (ctypes handle value)
    world: int
    rank: int
    rows: int            # rows reserved per rank (>= the largest local batch)
    gather_logits: bool = False


GATHERED_FIELDS = ("pred_vertices", "pred_keypoints_3d", "pred_keypoints_2d", "pred_cam", "pred_cam_t", "focal_length",
                   "rotmats", "betas")


class SmplOutput(NamedTuple):
    """The fields of the reference SMPL.forward output (smpl_wrapper.py:27-41) that its callers read."""
    vertices: torch.Tensor   # (B, V, 3)
    joints: torch.Tensor     # (B, 25 + n_extra, 3): 25 OpenPose joints + the regressed extra joints


class _SmplFacade:
    """`model.smpl`: `.faces` is read by demo.py:52; `model.smpl(global_orient=, body_pose=, betas=)` is the reference
    SMPL wrapper's forward on rotation matrices, differentiable in all three (SMPLifyInv, tokenhmr_b200.fitting)."""

    def __init__(self, model: SMPLModel):
        self._model = model
        self.faces = model.faces

    def __call__(self, global_orient: torch.Tensor, body_pose: torch.Tensor, betas: torch.Tensor,
                 pose2rot: bool = False) -> SmplOutput:
        """global_orient (B,1,3,3), body_pose (B,23,3,3), betas (B,nb), CUDA fp32.  pose2rot is ignored, as the
        reference's SMPLLayer ignores it (tokenhmr.py:176): the inputs are always rotation matrices."""
        verts, joints = self._model.forward(global_orient, body_pose, betas)
        return SmplOutput(verts, joints)


class TokenHMREngine(nn.Module):
    def __init__(self, cfg: TokenHMRConfig, state_dict: Dict[str, torch.Tensor], smpl: Dict[str, torch.Tensor],
                 device: str | torch.device = "cuda:0", max_batch: int = 256, use_cuda_graph: bool = True,
                 strict: bool = False, alias_outputs: bool = False, max_cached_shapes: int = 6,
                 concurrent: bool = False, fp8: bool = False):
        """strict: every contraction of the path in split-fp16 (3 tensor-core products, ~2^-21 relative: fp32-grade)
        instead of fp16 operands -- the mode whose results match the fp32 reference to 1e-4 with identical pose tokens
        (DESIGN.md §2); about 4x slower.  alias_outputs: return views of the engine's static output buffers (valid until
        the next forward of the same batch size / slot) instead of fresh tensors; TokenHMRPipeline uses it.
        max_batch: largest batch a forward accepts (bounds the workspace).  max_cached_shapes: distinct (batch size, slot)
        buffer sets kept alive; the least recently used one is dropped beyond that.
        concurrent: the forwards of different slots may run at the same time on different streams
        (TokenHMRPipeline(streams=2)); the engine then avoids kernels that need the whole GPU to themselves
        (thmr_config::concurrent).
        fp8: the ViT's QKV, fc1 and fc2 GEMMs (88 % of the model's FLOPs) run on block-scaled e4m3 operands on the FP8
        tensor cores (thmr_config::fp8, DESIGN.md §2 for its accuracy); not with strict.
        cfg.head selects the SMPL head: "token" (TokenHMR) or "transformer_decoder" (HMR 2.0's regression head, whose
        output dict has no cls_logits_softmax, as in the reference's forward_step, tokenhmr.py:157-158)."""
        if strict and fp8:
            raise _lib.ThmrError("strict and fp8 are exclusive numeric modes")
        super().__init__()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.ThmrError("TokenHMREngine needs a CUDA device (there is no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        lib()  # fail now if the shared library is missing
        from .checkpoint import validate_against_weights
        validate_against_weights(cfg, state_dict, smpl)
        self.strict = bool(strict)
        self.concurrent = bool(concurrent)
        self.fp8 = bool(fp8)
        self.has_logits = cfg.head == "token"     # the regression head has no token classifier
        self.alias_outputs = bool(alias_outputs)
        self.max_cached_shapes = int(max_cached_shapes)
        with torch.cuda.device(self.device):
            self.weights = PackedWeights(state_dict, cfg, self.device, strict=self.strict, fp8=self.fp8)
            self.smpl_model = SMPLModel(smpl, self.device)
            self.smpl = _SmplFacade(self.smpl_model)
            self._cfg_struct = make_config_struct(cfg, strict=self.strict, concurrent=self.concurrent,
                                                  fp8=self.fp8)
            h = ctypes.c_void_p()
            head = _lib.HEAD_TOKEN if self.has_logits else _lib.HEAD_REGRESSION
            check(lib().thmr_engine_create_head(ctypes.byref(self._cfg_struct), head, ctypes.byref(self.weights.struct),
                                                self.smpl_model.handle, ctypes.byref(h)))
            self._h = h
        self.max_batch = max_batch
        self.use_cuda_graph = use_cuda_graph
        self._bufs: Dict[int, dict] = {}     # per batch size: static buffers, workspace, optional graph
        self._dummy = nn.Parameter(torch.zeros(1), requires_grad=False)  # so .to()/.eval() behave like a Module

    # ------------------------------------------------------------------------------------------
    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().thmr_engine_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def to(self, *args, **kwargs):
        """The packed weights live on the device given at construction: `.to(that device)` (demo.py:35, eval.py:52) is a
        no-op, any other device or a dtype change raises instead of being silently ignored."""
        dev, dtype = None, kwargs.get("dtype")
        for a in list(args) + [kwargs.get("device")]:
            if isinstance(a, (str, torch.device, int)) and not isinstance(a, bool):
                dev = torch.device("cuda", a) if isinstance(a, int) else torch.device(a)
            elif isinstance(a, torch.dtype):
                dtype = a
            elif isinstance(a, torch.Tensor):
                dev, dtype = a.device, a.dtype
        if dev is not None:
            if dev.type == "cuda" and dev.index is None:
                dev = torch.device("cuda", torch.cuda.current_device())
            if dev != self.device:
                raise _lib.ThmrError(f"TokenHMREngine lives on {self.device}; .to({dev}) is not supported "
                                     "(build a new engine on that device; there is no CPU path)")
        if dtype is not None and dtype != torch.float32:
            raise _lib.ThmrError(f".to({dtype}): the engine's numeric contract is fixed (fp32 in / fp32 out)")
        return self

    def cpu(self):
        return self.to("cpu")

    def cuda(self, device=None):
        return self.to(torch.device("cuda", torch.cuda.current_device() if device is None else
                                    (device if isinstance(device, int) else torch.device(device).index or 0)))

    def half(self):
        return self.to(torch.float16)

    def num_launches(self) -> int:
        return lib().thmr_engine_num_launches(self._h)

    def _state(self, B: int, taps: bool, slot: int = 0, shard: Optional[ShardSpec] = None) -> dict:
        if B > self.max_batch:
            raise _lib.ThmrError(f"batch of {B} images exceeds max_batch={self.max_batch} (raise it at construction)")
        if shard is not None and not (0 < B <= shard.rows and 0 <= shard.rank < shard.world):
            raise _lib.ThmrError(f"shard {shard} cannot hold a local batch of {B}")
        if shard is not None and shard.gather_logits and not self.has_logits:
            raise _lib.ThmrError("gather_logits: a regression-head engine produces no cls_logits_softmax")
        key = (B, int(taps), slot) + ((shard.world, shard.rank, shard.rows, shard.gather_logits) if shard else ())
        st = self._bufs.get(key)
        if st is not None:
            self._bufs[key] = self._bufs.pop(key)          # most recently used last
            return st
        while len(self._bufs) >= max(1, self.max_cached_shapes):
            # drop the least recently used buffer set (its workspace, outputs and graph); the engine's plan cache is
            # keyed on the workspace pointer, so forget it if it pointed there
            old_key = next(iter(self._bufs))
            torch.cuda.synchronize(self.device)
            self._bufs.pop(old_key)
        c, dev = self.cfg, self.device
        nj = 25 + self.smpl_model.n_extra
        f = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        t = {
            "img": f(B, 3, c.image_size, c.image_size),
            **({"cls_logits_softmax": f(B, c.token_num, c.token_class_num)} if self.has_logits else {}),
            "pred_cam": f(B, 3), "rotmats": f(B, c.num_joints, 3, 3), "betas": f(B, c.num_betas),
            "pred_cam_t": f(B, 3), "focal_length": f(B, 2), "pred_keypoints_3d": f(B, nj, 3),
            "pred_vertices": f(B, self.smpl_model.num_verts, 3), "pred_keypoints_2d": f(B, nj, 2),
        }
        if taps:
            t.update({"vit_tokens": f(B, c.num_tokens, c.vit_dim), "token_out": f(B, c.dec_dim), "pose6d": f(B, 144)})
        g, gouts = None, None
        if shard is not None:
            # in-place all-gather layout: one buffer of world * rows images per gathered field; the engine writes this
            # rank's images straight into its rows (no pack / unpack copies)
            g, gouts = {}, _lib.Outputs()
            fields = GATHERED_FIELDS + (("cls_logits_softmax",) if shard.gather_logits else ())
            for name in fields:
                g[name] = f(shard.world * shard.rows, *t[name].shape[1:])
                t[name] = g[name][shard.rank * shard.rows: shard.rank * shard.rows + B]
                setattr(gouts, name, g[name].data_ptr())
        outs = _lib.Outputs()
        for name, _ in _lib.Outputs._fields_:
            if name in t:
                setattr(outs, name, t[name].data_ptr())
        nbytes = lib().thmr_engine_workspace_bytes(self._h, B)
        ws = torch.empty(nbytes + 1024, device=dev, dtype=torch.uint8)
        off = (-ws.data_ptr()) % 1024
        st = {"t": t, "outs": outs, "ws": ws, "ws_ptr": ws.data_ptr() + off, "graph": None, "warm": False,
              "g": g, "gouts": gouts, "shard": shard}
        self._bufs[key] = st
        return st

    def _launch(self, st: dict, B: int) -> None:
        stream = torch.cuda.current_stream().cuda_stream
        check(lib().thmr_engine_forward(self._h, st["t"]["img"].data_ptr(), B, ctypes.byref(st["outs"]), st["ws_ptr"],
                                        stream))
        sh = st["shard"]
        if sh is not None and sh.world > 1:
            # the one exchange of the sharded path: grouped in-place ncclAllGather, same stream (and same CUDA graph)
            check(lib().thmr_allgather_outputs(self._h, sh.comm, ctypes.byref(st["gouts"]), sh.rows, stream))

    @torch.no_grad()
    def forward(self, batch: Dict, return_taps: bool = False, slot: int = 0, alias_outputs: Optional[bool] = None,
                shard: Optional[ShardSpec] = None) -> Dict:
        """TokenHMR.forward: only batch['img'] is read (tokenhmr.py:146).  `slot` selects an independent set of
        input / output / workspace buffers (and CUDA graph), so that a caller can have several forwards in flight
        (TokenHMRPipeline).  Like the reference, the returned tensors are fresh (safe to keep across calls) unless
        alias_outputs is set, in which case they are views of that slot's buffers until its next forward
        (with `shard`: the gathered fields cover all world * rows images, see tokenhmr_b200.dist)."""
        alias = self.alias_outputs if alias_outputs is None else alias_outputs
        img = batch["img"]
        if img.dim() != 4 or img.shape[1] != 3 or img.shape[2] != self.cfg.image_size or img.shape[3] != self.cfg.image_size:
            raise _lib.ThmrError(f"batch['img'] must be (B,3,{self.cfg.image_size},{self.cfg.image_size}), got {tuple(img.shape)}")
        B = img.shape[0]
        with torch.cuda.device(self.device):
            st = self._state(B, return_taps, slot, shard)
            st["t"]["img"].copy_(img.to(torch.float32), non_blocking=True)     # H2D (or D2D) of the batch
            if self.use_cuda_graph:
                if st["graph"] is None:
                    if not st["warm"]:
                        self._launch(st, B)       # eager call builds the plans and configures the kernels
                        torch.cuda.current_stream().synchronize()
                        st["warm"] = True
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        self._launch(st, B)
                    st["graph"] = g
                st["graph"].replay()
            else:
                self._launch(st, B)
            t = dict(st["t"])
            if st["g"] is not None:
                t.update(st["g"])           # gathered fields: all world * rows images
            rot = t["rotmats"]
            out = {
                **({"cls_logits_softmax": t["cls_logits_softmax"]} if self.has_logits else {}),
                "pred_cam": t["pred_cam"],
                "pred_smpl_params": {"global_orient": rot[:, :1].clone(), "body_pose": rot[:, 1:].clone(),
                                     "betas": t["betas"].clone()},
                "pred_cam_t": t["pred_cam_t"],
                "focal_length": t["focal_length"],
                "pred_keypoints_3d": t["pred_keypoints_3d"],
                "pred_vertices": t["pred_vertices"],
                "pred_keypoints_2d": t["pred_keypoints_2d"],
            }
            if return_taps:
                out["_vit_tokens"], out["_token_out"], out["_pred_body_pose_6d"] = t["vit_tokens"], t["token_out"], t["pose6d"]
            if not alias:
                out = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}
        return out

    @torch.no_grad()
    def profile(self, img: torch.Tensor) -> list:
        """One eager forward with a CUDA event between launch groups.  Returns [(label, ms, flops, bytes), ...]
        (labels and algorithmic work come from the engine: thmr_engine_step_info)."""
        B = img.shape[0]
        with torch.cuda.device(self.device):
            st = self._state(B, False)
            st["t"]["img"].copy_(img.to(torch.float32))
            if not st["warm"]:
                self._launch(st, B)
                torch.cuda.current_stream().synchronize()
                st["warm"] = True
            n = lib().thmr_engine_num_steps(self._h)
            ms = (ctypes.c_float * n)()
            check(lib().thmr_engine_profile(self._h, st["t"]["img"].data_ptr(), B, ctypes.byref(st["outs"]),
                                            st["ws_ptr"], torch.cuda.current_stream().cuda_stream, ms, n))
            out = []
            for i in range(n):
                name, fl, by = ctypes.c_char_p(), ctypes.c_double(), ctypes.c_double()
                check(lib().thmr_engine_step_info(self._h, i, ctypes.byref(name), ctypes.byref(fl), ctypes.byref(by)))
                out.append((name.value.decode(), float(ms[i]), fl.value, by.value))
            return out

    @torch.no_grad()
    def profile_in_graph(self, img: torch.Tensor, replays: int = 20) -> list:
        """Per-step device time INSIDE the CUDA-graph replay: every kernel of the forward stamps the GPU's nanosecond timer
        when it starts (thmr_engine_forward_stamped); `replays` back-to-back replays of that graph keep the chip in its
        sustained state and the stamps of the last one are read.  Returns [(label, ms, flops, bytes), ...] like profile();
        a step without a stamped kernel reports 0 and its time is part of the step before it.  The entries sum to the
        replay's duration: unlike the event-separated profile() nothing is inserted between the launches."""
        B = img.shape[0]
        with torch.cuda.device(self.device):
            st = self._state(B, False, slot=-1)
            st["t"]["img"].copy_(img.to(torch.float32))
            stream = lambda: torch.cuda.current_stream().cuda_stream
            launch = lambda: check(lib().thmr_engine_forward_stamped(self._h, st["t"]["img"].data_ptr(), B,
                                                                     ctypes.byref(st["outs"]), st["ws_ptr"], stream()))
            if st["graph"] is None:
                launch()
                torch.cuda.current_stream().synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    launch()
                st["graph"] = g
            for _ in range(max(1, replays)):
                st["graph"].replay()
            torch.cuda.current_stream().synchronize()
            n = lib().thmr_engine_num_steps(self._h)
            buf = (ctypes.c_uint64 * (n + 1))()
            got = lib().thmr_engine_read_stamps(self._h, buf, n + 1)
            if got != n + 1:
                check(got if got < 0 else -1)
            t = [int(v) for v in buf]
            out, starts = [], [i for i in range(n) if t[i] != 0] + [n]
            dur = {i: 0.0 for i in range(n)}
            for a, b in zip(starts[:-1], starts[1:]):
                dur[a] = (t[b] - t[a]) * 1e-6
            for i in range(n):
                name, fl, by = ctypes.c_char_p(), ctypes.c_double(), ctypes.c_double()
                check(lib().thmr_engine_step_info(self._h, i, ctypes.byref(name), ctypes.byref(fl), ctypes.byref(by)))
                out.append((name.value.decode(), dur[i], fl.value, by.value))
            return out

    @torch.no_grad()
    def backbone(self, img: torch.Tensor) -> torch.Tensor:
        """ViT.forward (vit.py:341-343): (B,3,256,256) -> (B,1280,16,12) like the reference backbone."""
        B = img.shape[0]
        with torch.cuda.device(self.device):
            st = self._state(B, True)
            st["t"]["img"].copy_(img.to(torch.float32), non_blocking=True)
            check(lib().thmr_engine_vit_forward(self._h, st["t"]["img"].data_ptr(), B, st["t"]["vit_tokens"].data_ptr(),
                                                st["ws_ptr"], torch.cuda.current_stream().cuda_stream))
            tok = st["t"]["vit_tokens"]
            gh, gw = self.cfg.grid_h, self.cfg.grid_w
            return tok.permute(0, 2, 1).reshape(B, self.cfg.vit_dim, gh, gw).contiguous()


class TokenHMRPipeline:
    """Double-buffered host -> device -> host driver for streams of batches (eval.py / track.py style loops):

        pipe = TokenHMRPipeline(model, read_back=("pred_vertices", "pred_keypoints_3d", "pred_cam", "pred_cam_t"))
        t0 = pipe.submit(batch0)            # H2D of the pinned host batch on the copy stream, forward, D2H: all async
        t1 = pipe.submit(batch1)            # its H2D overlaps the forward of batch0
        out0 = pipe.result(t0)              # pinned host tensors (valid until the slot is reused, `depth` submits later)

    Nothing is skipped: every submit copies its own input and every result is read back; only the waiting is moved, so
    the copy engines work while the SMs run the previous batch.  `post(out)` (optional) runs on the compute stream between
    the forward and the read-back (e.g. the all-gather of a sharded model).

    streams=2 additionally lets the forwards of consecutive batches overlap on the SMs: slot s replays its CUDA graph
    on compute stream s % streams, so the latency-bound tail of batch i (token decoder, classifier, tokenizer decoder,
    SMPL: ~80 small launches that leave most SMs idle) runs under the ViT GEMMs of batch i+1.  Needs an engine built
    with concurrent=True; single-GPU only (the sharded forward's in-graph collective keeps one stream)."""

    def __init__(self, model: "TokenHMREngine", depth: int = 2, read_back=("pred_vertices", "pred_keypoints_3d",
                                                                         "pred_cam", "pred_cam_t"), post=None,
                 shard: Optional[ShardSpec] = None, read_rows: Optional[slice] = None, streams: int = 1):
        """shard: run every forward as this rank's part of a sharded batch (in-place all-gather inside the forward's CUDA
        graph).  read_rows: rows of each output to copy back to the host (e.g. only this rank's own images when the
        ranks of one host each hand their shard to the same consumer); default all rows."""
        self.model, self.depth, self.read_back, self.post = model, int(depth), tuple(read_back), post
        self.shard, self.read_rows = shard, read_rows
        self.streams = int(streams)
        if not 1 <= self.streams <= self.depth:
            raise _lib.ThmrError(f"TokenHMRPipeline: streams={streams} must be in [1, depth={depth}]")
        if self.streams > 1 and not getattr(model, "concurrent", False):
            raise _lib.ThmrError("TokenHMRPipeline(streams > 1) needs TokenHMREngine(concurrent=True)")
        if self.streams > 1 and shard is not None and shard.world > 1:
            raise _lib.ThmrError("TokenHMRPipeline(streams > 1): the sharded forward (in-graph collective) keeps one stream")
        with torch.cuda.device(model.device):
            self.copy_stream = torch.cuda.Stream(model.device)
            self.compute_streams = [torch.cuda.Stream(model.device) for _ in range(self.streams)]
            self.compute_stream = self.compute_streams[0]
            self._copied = [torch.cuda.Event() for _ in range(self.depth)]
            self._done = [torch.cuda.Event() for _ in range(self.depth)]
        self._used = [False] * self.depth
        self._host = [dict() for _ in range(self.depth)]
        self._n = 0

    @torch.no_grad()
    def submit(self, batch: Dict) -> int:
        ticket = self._n
        slot = ticket % self.depth
        self._n += 1
        m = self.model
        img = batch["img"]
        with torch.cuda.device(m.device):
            st = m._state(img.shape[0], False, slot, self.shard)
            with torch.cuda.stream(self.copy_stream):
                if self._used[slot]:
                    self.copy_stream.wait_event(self._done[slot])       # the slot's previous forward has consumed its input
                st["t"]["img"].copy_(img, non_blocking=True)
                self._copied[slot].record(self.copy_stream)
            cs = self.compute_streams[slot % self.streams]
            with torch.cuda.stream(cs):
                cs.wait_event(self._copied[slot])
                out = m.forward({"img": st["t"]["img"]}, slot=slot, alias_outputs=True,   # (input self-copy: a no-op)
                                shard=self.shard)
                if self.post is not None:
                    out = self.post(out)
                host = self._host[slot]
                for k in self.read_back:
                    src = out[k] if self.read_rows is None else out[k][self.read_rows]
                    if k not in host or host[k].shape != src.shape:
                        host[k] = torch.empty(src.shape, dtype=src.dtype).pin_memory()
                    host[k].copy_(src, non_blocking=True)
                self._done[slot].record(cs)
            self._used[slot] = True
        return ticket

    def join(self) -> "torch.cuda.Stream":
        """compute_stream after it has been made to wait for every submitted batch (all slots, all streams): the place
        to record an end-of-work event."""
        for used, ev in zip(self._used, self._done):
            if used:
                self.compute_stream.wait_event(ev)
        return self.compute_stream

    def result(self, ticket: int) -> Dict[str, torch.Tensor]:
        slot = ticket % self.depth
        self._done[slot].synchronize()
        return self._host[slot]


def load_tokenhmr(state_dict: Dict[str, torch.Tensor], smpl: Dict[str, torch.Tensor],
                  cfg: Optional[TokenHMRConfig] = None, device: str = "cuda:0", **kw):
    """Counterpart of lib.models.load_tokenhmr (tokenhmr/lib/models/__init__.py:3-26): returns (model, cfg).
    `state_dict` uses the reference key names (see tokenhmr_b200.weights.strip_checkpoint)."""
    cfg = cfg or TokenHMRConfig()
    model = TokenHMREngine(cfg, state_dict, smpl, device=device, **kw)
    return model, cfg
