"""The PointNav policy step on the library's kernels: depth in -> action, with each environment's hidden state and previous
action updated in place.

Encoder: every conv is an im2col pass (``vlfm_pointnav_depth_in`` for conv1, ``vlfm_sam_im2col3x3`` for the 3x3 convs,
``vlfm_pointnav_gather_s2`` for the stride-2 1x1 downsamples) plus the wgmma GEMM (fp16 operands, fp32 out) through
``vlm/dense.py``; each GroupNorm, with the block's residual add (identity, or the downsample's GroupNorm) and ReLU, is one
``vlfm_pointnav_groupnorm`` launch on the fp32 GEMM output.  Recurrent part in fp32: ``visual_fc`` (weight columns permuted
from the NCHW flatten to NHWC), the two LSTM gate GEMMs ([x | h] @ [W_ih | W_hh]^T + b_ih + b_hh) on
``vlfm_pointnav_gemv_f32``, the cells and the head on ``vlfm_pointnav_lstm_*``.

The step for a batch size and frame size is captured in a CUDA graph on its first call and replayed after; every launch is
deterministic, so a replay is bitwise equal to an eager run.  An environment's result does not depend on the batch it shares,
except through the conv GEMMs, whose row tiling depends on the batch size.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import torch

from .. import _lib
from ..vlm.dense import gemm_f16
from .pointnav_weights import BACKBONE, EMB, HEAD_CONTINUOUS, HEAD_DISCRETE, HID, NGROUPS, STAGES, VIS

F16, F32 = torch.float16, torch.float32
GN_EPS = 1e-5
LD0 = VIS + 2 * EMB + HID     # layer-0 GEMV input row [visual | goal | prev action | h_l0]
LD1 = 2 * HID                 # layer-1 GEMV input row [h_l0' | h_l1]
MAX_GEMV_BATCH = 64


def _half(n: int) -> int:
    """output side of a stride-2 conv with pad 1 (3x3) or pad 0 (1x1), and of the 3x3 stride-2 pad-1 max pool"""
    return (n - 1) // 2 + 1


def spatial_plan(hw: Tuple[int, int]) -> List[Tuple[int, int]]:
    """Map sizes: [pooled input, conv1, maxpool / layer1, layer2, layer3, layer4]; raises unless the final map is 4 x 4."""
    h, w = hw[0] // 2, hw[1] // 2
    if h < 1 or w < 1:
        raise ValueError(f"PointNav: input size {hw} too small")
    sizes = [(h, w)]
    for _ in range(2):          # conv1 (stride 2), max pool (stride 2)
        h, w = _half(h), _half(w)
        sizes.append((h, w))
    for _, stride in STAGES[1:]:
        h, w = _half(h), _half(w)
        sizes.append((h, w))
    if (h, w) != (4, 4):
        raise ValueError(f"PointNav: input size {hw} gives a {h} x {w} final map; visual_fc needs 4 x 4 (224 x 224 and 212 x 240 do)")
    return sizes


def conv_rows(w: torch.Tensor) -> torch.Tensor:
    """[O, C, k, k] -> [O, ldk] fp16 GEMM rows with columns (ky, kx, c), K zero-padded to a multiple of 8."""
    O, C, k, _ = w.shape
    r = w.permute(0, 2, 3, 1).reshape(O, k * k * C)
    ldk = (k * k * C + 7) // 8 * 8
    return torch.nn.functional.pad(r, (0, ldk - r.shape[1])).to(F16).contiguous()


class PointNavEngine:
    def __init__(self, w: Dict[str, torch.Tensor], discrete: bool, max_batch: int = 1, input_hw: Tuple[int, int] = (224, 224),
                 num_envs: Optional[int] = None, device="cuda", use_graph: bool = True) -> None:
        if not torch.cuda.is_available():
            raise _lib.VlfmError("vlfm_b200 needs a CUDA device (no CPU fallback)")
        if not 1 <= max_batch <= MAX_GEMV_BATCH:
            raise ValueError(f"PointNav: max_batch must be in [1, {MAX_GEMV_BATCH}], got {max_batch}")
        self.lib = _lib.load()
        self.dev = torch.device(device)
        self.discrete, self.max_batch, self.input_hw = discrete, max_batch, tuple(input_hw)
        self.num_envs = num_envs or max_batch
        self.sizes = spatial_plan(self.input_hw)
        self.use_graph = use_graph and os.environ.get("VLFM_NO_GRAPH", "") != "1"
        dev = self.dev
        f = lambda t: t.to(dev, F32).contiguous()
        self.w: Dict[str, torch.Tensor] = {}
        for k, v in w.items():
            if v.dim() == 4:
                self.w[k] = conv_rows(v).to(dev)
            elif not k.startswith("net.state_encoder.") and k != "net.visual_fc.1.weight":
                self.w[k] = f(v)
        # visual_fc over the NHWC flatten: column (y*4 + x)*128 + c holds the reference's column c*16 + y*4 + x
        vw = w["net.visual_fc.1.weight"].reshape(VIS, 128, 4, 4).permute(0, 2, 3, 1).reshape(VIS, 2048)
        self.w["net.visual_fc.1.weight"] = f(vw)
        rnn = "net.state_encoder.rnn."
        for l in range(2):
            self.w[f"lstm{l}.w"] = f(torch.cat([w[f"{rnn}weight_ih_l{l}"], w[f"{rnn}weight_hh_l{l}"]], 1))
            self.w[f"lstm{l}.b"] = f(w[f"{rnn}bias_ih_l{l}"].double() + w[f"{rnn}bias_hh_l{l}"].double())
        head = HEAD_DISCRETE if discrete else HEAD_CONTINUOUS
        self.w["head.w"], self.w["head.b"] = self.w[head + "weight"], self.w[head + "bias"]

        # per-environment state: [h_l0, h_l1, c_l0, c_l1] and the previous action
        E = self.num_envs
        self.hidden = torch.zeros(E, 4, HID, dtype=F32, device=dev)
        self.prev = torch.zeros(E, 1, dtype=torch.long, device=dev) if discrete else torch.zeros(E, 2, dtype=F32, device=dev)
        # step inputs / outputs
        B = max_batch
        self.goal = torch.zeros(B, 2, dtype=F32, device=dev)
        self.masks = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.env_ids = torch.zeros(B, dtype=torch.int32, device=dev)
        self.action = torch.zeros(B, 1, dtype=torch.long, device=dev) if discrete else torch.zeros(B, 2, dtype=F32, device=dev)
        self.head = torch.zeros(B, 4, dtype=F32, device=dev)
        self.features = torch.zeros(B, HID, dtype=F32, device=dev)
        self.visual = torch.zeros(B, 2048, dtype=F32, device=dev)
        self.xin0 = torch.zeros(B, LD0, dtype=F32, device=dev)
        self.xin1 = torch.zeros(B, LD1, dtype=F32, device=dev)
        self.cbuf = torch.zeros(B, 2 * HID, dtype=F32, device=dev)
        self.gates = torch.zeros(B, 4 * HID, dtype=F32, device=dev)
        # encoder scratch, sized by the largest stage at max_batch
        (ph, pw), (h1, w1), (h2, w2) = self.sizes[0], self.sizes[1], self.sizes[2]
        col = B * h1 * w1 * 56
        act = B * h1 * w1 * 32
        hw, cin = (h2, w2), 32
        for (c, _), (h, ww) in zip(STAGES, self.sizes[2:]):
            col = max(col, B * h * ww * 9 * max(cin, c))
            act = max(act, B * h * ww * c, B * hw[0] * hw[1] * cin)
            hw, cin = (h, ww), c
        col = max(col, B * 16 * 9 * 256)
        self.col = torch.empty(col, dtype=F16, device=dev)
        self.t32 = torch.empty(act, dtype=F32, device=dev)
        self.d32 = torch.empty(act, dtype=F32, device=dev)
        self.x32 = torch.empty(act, dtype=F32, device=dev)
        self.x16 = torch.empty(act, dtype=F16, device=dev)
        self.t16 = torch.empty(act, dtype=F16, device=dev)
        self.g16 = torch.empty(act, dtype=F16, device=dev)
        self._graphs: Dict[Tuple[int, int, int], Tuple[torch.cuda.CUDAGraph, torch.Tensor]] = {}

    # ---------------------------------------------------------------------------------------------------------- launches
    def _gemm(self, a_buf, M, K, wname, out_buf, N):
        gemm_f16(a_buf[:M * K].view(M, K), self.w[wname], None, _lib.EPI_BIAS_F32, out=out_buf[:M * N].view(M, N))

    def _gn(self, x, name, B, HW, C, G, rmode=0, r=None, y=None, name_b=None, out32=None, out16=None, relu=1):
        gb, bb = (self.w[name_b + ".weight"].data_ptr(), self.w[name_b + ".bias"].data_ptr()) if name_b else (None, None)
        rc = self.lib.vlfm_pointnav_groupnorm(x.data_ptr(), self.w[name + ".weight"].data_ptr(), self.w[name + ".bias"].data_ptr(), rmode,
                                              _lib.ptr(r), _lib.ptr(y), gb, bb, _lib.ptr(out32), _lib.ptr(out16), B, HW, C, G, GN_EPS,
                                              relu, _lib.stream_ptr())
        _lib.check(rc, "vlfm_pointnav_groupnorm")

    def _im2col(self, x16, B, H, W, C, stride):
        rc = self.lib.vlfm_sam_im2col3x3(x16.data_ptr(), self.col.data_ptr(), B, H, W, C, stride, 9 * C, _lib.stream_ptr())
        _lib.check(rc, "vlfm_sam_im2col3x3")

    def _gemv(self, x, ldx, wname, bname, y, ldy, B, N, K, relu):
        rc = self.lib.vlfm_pointnav_gemv_f32(x.data_ptr(), ldx, self.w[wname].data_ptr(), self.w[wname].shape[1], self.w[bname].data_ptr(),
                                             y.data_ptr(), ldy, B, N, K, relu, _lib.stream_ptr())
        _lib.check(rc, "vlfm_pointnav_gemv_f32")

    def _forward(self, depth: torch.Tensor) -> None:
        B, H, W = depth.shape
        IH, IW = self.input_hw
        st = _lib.stream_ptr()
        (h1, w1), (h, w) = self.sizes[1], self.sizes[2]
        # stem: resize + pool + conv1 rows, GEMM, GroupNorm + ReLU, max pool
        _lib.check(self.lib.vlfm_pointnav_depth_in(depth.data_ptr(), B, H, W, IH, IW, self.col.data_ptr(), 56, None, st),
                   "vlfm_pointnav_depth_in")
        M = B * h1 * w1
        self._gemm(self.col, M, 56, BACKBONE + "conv1.0.weight", self.t32, 32)
        self._gn(self.t32, BACKBONE + "conv1.1", B, h1 * w1, 32, NGROUPS, out32=self.d32)
        _lib.check(self.lib.vlfm_pointnav_maxpool3s2(self.d32.data_ptr(), self.x32.data_ptr(), self.x16.data_ptr(), B, h1, w1, 32, st),
                   "vlfm_pointnav_maxpool3s2")
        cin = 32
        for li, ((c, stride), (ho, wo)) in enumerate(zip(STAGES, self.sizes[2:]), start=1):
            for bi in range(2):
                p = f"{BACKBONE}layer{li}.{bi}."
                s = stride if bi == 0 else 1
                ci = cin if bi == 0 else c
                M = B * ho * wo
                self._im2col(self.x16, B, h, w, ci, s)
                self._gemm(self.col, M, 9 * ci, p + "convs.0.weight", self.t32, c)
                self._gn(self.t32, p + "convs.1", B, ho * wo, c, NGROUPS, out16=self.t16)
                self._im2col(self.t16, B, ho, wo, c, 1)
                self._gemm(self.col, M, 9 * c, p + "convs.3.weight", self.t32, c)
                if p + "downsample.0.weight" in self.w:
                    _lib.check(self.lib.vlfm_pointnav_gather_s2(self.x16.data_ptr(), self.g16.data_ptr(), B, h, w, ci, st), "vlfm_pointnav_gather_s2")
                    self._gemm(self.g16, M, ci, p + "downsample.0.weight", self.d32, c)
                    self._gn(self.t32, p + "convs.4", B, ho * wo, c, NGROUPS, rmode=2, y=self.d32, name_b=p + "downsample.1",
                             out32=self.x32, out16=self.x16)
                else:
                    self._gn(self.t32, p + "convs.4", B, ho * wo, c, NGROUPS, rmode=1, r=self.x32, out32=self.x32, out16=self.x16)
                h, w = ho, wo
            cin = c
        # compression conv + GroupNorm(1) + ReLU -> the NHWC flatten [B, 2048]
        self._im2col(self.x16, B, 4, 4, 256, 1)
        self._gemm(self.col, B * 16, 9 * 256, "net.visual_encoder.compression.0.weight", self.t32, 128)
        self._gn(self.t32, "net.visual_encoder.compression.1", B, 16, 128, 1, out32=self.visual)
        # recurrent part (fp32)
        wp = self.w["net.prev_action_embedding.weight"]
        bp = self.w.get("net.prev_action_embedding.bias")
        rc = self.lib.vlfm_pointnav_lstm_prep(self.env_ids.data_ptr(), self.hidden.data_ptr(), self.prev.data_ptr(), int(self.discrete),
                                              self.masks.data_ptr(), self.goal.data_ptr(), self.w["net.tgt_embeding.weight"].data_ptr(),
                                              self.w["net.tgt_embeding.bias"].data_ptr(), wp.data_ptr(), _lib.ptr(bp), self.xin0.data_ptr(),
                                              self.xin1.data_ptr(), self.cbuf.data_ptr(), B, st)
        _lib.check(rc, "vlfm_pointnav_lstm_prep")
        self._gemv(self.visual, 2048, "net.visual_fc.1.weight", "net.visual_fc.1.bias", self.xin0, LD0, B, VIS, 2048, 1)
        self._gemv(self.xin0, LD0, "lstm0.w", "lstm0.b", self.gates, 4 * HID, B, 4 * HID, LD0, 0)
        _lib.check(self.lib.vlfm_pointnav_lstm_cell(self.gates.data_ptr(), self.cbuf.data_ptr(), self.xin1.data_ptr(), B, st),
                   "vlfm_pointnav_lstm_cell")
        self._gemv(self.xin1, LD1, "lstm1.w", "lstm1.b", self.gates, 4 * HID, B, 4 * HID, LD1, 0)
        rc = self.lib.vlfm_pointnav_lstm_head(self.gates.data_ptr(), self.cbuf.data_ptr(), self.xin1.data_ptr(), self.w["head.w"].data_ptr(),
                                              self.w["head.b"].data_ptr(), int(self.discrete), self.env_ids.data_ptr(), self.hidden.data_ptr(),
                                              self.prev.data_ptr(), self.features.data_ptr(), self.head.data_ptr(), self.action.data_ptr(), B, st)
        _lib.check(rc, "vlfm_pointnav_lstm_head")

    # ------------------------------------------------------------------------------------------------------------- step
    @torch.inference_mode()
    def step(self, depth: torch.Tensor, goal: torch.Tensor, masks: torch.Tensor, env_ids: torch.Tensor, graph: Optional[bool] = None) -> None:
        """depth [B,H,W] fp32 (device, any frame size), goal [B,2], masks [B] bool, env_ids [B] int (distinct state slots).  Writes
        self.action / head / features [:B] and updates self.hidden / self.prev at env_ids.  ``graph=False`` runs eagerly."""
        B = depth.shape[0]
        key = (B, depth.shape[1], depth.shape[2])
        with torch.cuda.device(self.dev):
            self.goal[:B].copy_(goal, non_blocking=True)
            self.masks[:B].copy_(masks, non_blocking=True)
            self.env_ids[:B].copy_(env_ids, non_blocking=True)
            use_graph = self.use_graph if graph is None else graph
            if not use_graph:
                self._forward(depth.contiguous())
                return
            if key not in self._graphs:
                static_in = depth.contiguous().clone()
                self._forward(static_in)          # this call's step, eagerly; it also sets the kernels' attributes
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):          # capture records the launches without running them
                    self._forward(static_in)
                self._graphs[key] = (g, static_in)
                return
            g, static_in = self._graphs[key]
            static_in.copy_(depth, non_blocking=True)
            g.replay()

    def launches_per_step(self, B: int = 1, hw: Optional[Tuple[int, int]] = None) -> int:
        """Kernels one step launches (counted on an eager run that leaves the state unchanged)."""
        hw = hw or self.input_hw
        saved = (self.hidden.clone(), self.prev.clone())
        depth = torch.zeros(B, *hw, dtype=F32, device=self.dev)
        zeros = torch.zeros(B, dtype=torch.bool, device=self.dev)
        n0 = _lib.launch_count()
        self.step(depth, torch.zeros(B, 2, device=self.dev), zeros, torch.arange(B, device=self.dev), graph=False)
        n = _lib.launch_count() - n0
        self.hidden.copy_(saved[0])
        self.prev.copy_(saved[1])
        return n
