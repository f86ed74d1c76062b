"""YOLOv7 on the library's kernels: a layer plan built from the module tree, activations in buffers shared by last use, and one
CUDA graph per (B, H, W) for preprocess + network + decode + NMS + box mapping.

Activations are fp16 NHWC rows.  A layer whose output feeds a Concat writes straight into its channel slice of the concat's
buffer (GEMM ``ldo``, strided pools / upsample / add), so no Concat copies anything.  1x1 convs are GEMMs on the rows, 3x3 convs
``dense.im2col`` (its input may be a slice) plus the GEMM, all with the folded BatchNorm in the bias and SiLU in the epilogue.
Thresholds and the class filter sit in a device parameter block, so changing them does not re-capture.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _lib
from ..utils.cuda_graph import GraphCache, default_use_graph
from .dense import conv_rows, gemm_f16, im2col
from .yolov7_weights import Layer, fold, fold_detect

F16 = torch.float16
IN_H, IN_W = 448, 640          # cv2.resize(image, (640, int(640 * 0.7)))
MAX_DET = 300                  # yolov7 non_max_suppression max_det
MAX_NMS = 30000                # its max_nms: never reached (the network has fewer candidate rows)


def area_tables(ssize: int, dsize: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """cv2's computeResizeAreaTab (INTER_AREA, downscale) in CSR form: (ofs [dsize + 1], src index, weight float32), in double
    as cv2 computes them (scale = 1 / (dsize / ssize))."""
    scale = 1.0 / (dsize / ssize)
    ofs, si, al = [0], [], []
    for d in range(dsize):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, ssize - f1)
        s1, s2 = int(np.ceil(f1)), int(np.floor(f2))
        s2 = min(s2, ssize - 1)
        s1 = min(s1, s2)
        if s1 - f1 > 1e-3:
            si.append(s1 - 1); al.append(np.float32((s1 - f1) / cell))
        for s in range(s1, s2):
            si.append(s); al.append(np.float32(1.0 / cell))
        if f2 - s2 > 1e-3:
            si.append(s2); al.append(np.float32(min(min(f2 - s2, 1.0), cell) / cell))
        ofs.append(len(si))
    return np.asarray(ofs, np.int32), np.asarray(si, np.int32), np.asarray(al, np.float32)


def check_frame(H: int, W: int) -> None:
    """Frames the cv2 INTER_AREA restatement covers: downscales that are not integer on both axes (cv2 then takes its
    resizeAreaFast path), or the identity."""
    if H < IN_H or W < IN_W:
        raise ValueError(f"YOLOv7: frames must be at least {IN_W}x{IN_H} (got {W}x{H}); cv2 INTER_AREA upscales differently")
    if (H, W) != (IN_H, IN_W) and H % IN_H == 0 and W % IN_W == 0:
        raise NotImplementedError(f"YOLOv7: {W}x{H} is an integer downscale on both axes (cv2's resizeAreaFast path), not implemented")


def scale_coords_params(H: int, W: int) -> Tuple[float, float, float]:
    """yolov7 scale_coords((448, 640), boxes, (H, W)) treats the input as a letterbox of the frame: (gain, pad_x, pad_y)."""
    gain = min(IN_H / H, IN_W / W)
    return gain, (IN_W - W * gain) / 2, (IN_H - H * gain) / 2


@dataclass
class View:
    """A layer output: ``store`` (index of a buffer), channel offset, channels, row stride, spatial size."""
    store: int
    off: int
    c: int
    h: int
    w: int


class YoloEngine:
    def __init__(self, layers: List[Layer], device=None):
        self.dev = torch.device(device or "cuda")
        self.lib = _lib.load()
        self.layers = layers
        det = layers[-1]
        self.nc = int(det.extra["nc"])
        self.na = int(det.extra["anchors"].shape[1])
        self.no = self.nc + 5
        if self.nc > 128:
            raise NotImplementedError(f"YOLOv7: {self.nc} classes (at most 128)")
        self._fold_weights()
        self._plan()
        self.params = torch.zeros(8, dtype=torch.int32, device=self.dev)      # VlfmYoloParams
        self._bufs: Dict[int, dict] = {}
        self._tables: Dict[Tuple[int, int], tuple] = {}
        self.use_graph = default_use_graph()
        self.graphs = GraphCache()
        self.set_params(0.25, 0.45, None, False)

    # --------------------------------------------------------------------------------------------------------- weights
    def _fold_weights(self) -> None:
        self.w: Dict[Tuple[int, str], Tuple[torch.Tensor, torch.Tensor, int, int]] = {}
        det = self.layers[-1]
        for l in self.layers:
            for name, c in l.convs.items():
                if l.type == "Detect":
                    k = int(name[1:])
                    wf, bf = fold_detect(c, det.extra["ia"][k], det.extra["im"][k])
                else:
                    wf, bf = fold(c)
                if l.type == "Conv" and wf.shape[1] == 12 and l.f[0] >= 0 and self._is_reorg(l.f[0]):
                    wf = torch.nn.functional.pad(wf, (0, 0, 0, 0, 0, 4))      # ReOrg's map: 12 channels + 4 zero
                self.w[(l.i, name)] = (conv_rows(wf).to(self.dev, F16), bf.to(self.dev, torch.float32).contiguous(), wf.shape[2], c.stride)
        self.anchors = det.extra["anchors"].to(self.dev, torch.float32).reshape(-1, self.na, 2).contiguous()
        self.strides = [float(s) for s in det.extra["strides"]]

    def _is_reorg(self, i: int) -> bool:
        return any(l.i == i and l.type == "ReOrg" for l in self.layers)

    # ------------------------------------------------------------------------------------------------------------ plan
    def _plan(self) -> None:
        """Output views, concat placement and buffer sharing by last use (per image element counts; x B at allocation)."""
        by_i = {l.i: l for l in self.layers}
        if self.layers[0].type != "ReOrg" or self.layers[0].f != [-1]:
            raise NotImplementedError("YOLOv7: the network must start with ReOrg of the input")
        shape: Dict[int, Tuple[int, int, int]] = {}           # i -> (h, w, c)
        for l in self.layers:
            if l.type == "ReOrg":
                shape[l.i] = (IN_H // 2, IN_W // 2, 16)         # 12 channels + 4 zero (the first conv's K padding)
                continue
            h, w, c = shape[l.f[0]]
            if l.type == "Conv":
                cv = l.convs[""]
                s = cv.stride
                shape[l.i] = ((h - 1) // s + 1, (w - 1) // s + 1, cv.w.shape[0])
            elif l.type == "DownC":
                shape[l.i] = (h // 2, w // 2, l.convs["cv2"].w.shape[0] + l.convs["cv3"].w.shape[0])
            elif l.type == "SPPCSPC":
                shape[l.i] = (h, w, l.convs["cv7"].w.shape[0])
            elif l.type == "Upsample":
                shape[l.i] = (2 * h, 2 * w, c)
            elif l.type == "Concat":
                hw = {shape[j][:2] for j in l.f}
                if len(hw) != 1:
                    raise ValueError(f"YOLOv7: layer {l.i} concatenates maps of sizes {sorted(hw)}")
                shape[l.i] = (h, w, sum(shape[j][2] for j in l.f))
            elif l.type == "Shortcut":
                if len(l.f) != 2 or shape[l.f[0]] != shape[l.f[1]]:
                    raise ValueError(f"YOLOv7: layer {l.i} adds {[shape[j] for j in l.f]}")
                shape[l.i] = shape[l.f[0]]
            else:
                shape[l.i] = (0, 0, 0)
            if l.type in ("Conv", "DownC", "SPPCSPC"):
                cin = shape[l.f[0]][2]
                first = next(iter(l.convs.values()))
                if first.w.shape[1] != cin and not (cin == 16 and first.w.shape[1] == 12):
                    raise ValueError(f"YOLOv7: layer {l.i} ({l.type}) takes {first.w.shape[1]} channels, its input has {cin}")
        self.shape = shape
        # concat placement: each producer writes into the one concat that reads it
        place: Dict[int, Tuple[int, int]] = {}
        for l in self.layers:
            if l.type != "Concat":
                continue
            off = 0
            for j in l.f:
                p = by_i[j]
                if j in place or l.f.count(j) != 1 or p.type in ("ReOrg", "Concat", "Detect"):
                    raise NotImplementedError(f"YOLOv7: layer {l.i} concatenates layer {j} ({p.type}), which cannot write into it")
                place[j] = (l.i, off)
                off += shape[j][2]
        # storages: every non-placed layer owns one; lifetimes over plan positions
        pos = {l.i: n for n, l in enumerate(self.layers)}
        last = {l.i: pos[l.i] for l in self.layers}
        for l in self.layers:
            for j in l.f:
                if j >= 0:
                    last[j] = max(last[j], pos[l.i])
        self.views: Dict[int, View] = {}
        owner: Dict[int, int] = {}
        stores: List[List[int]] = []                              # [elements per image, first, last]
        for l in self.layers:
            if l.type == "Detect":
                continue
            h, w, c = shape[l.i]
            if l.i in place:
                continue
            owner[l.i] = len(stores)
            stores.append([h * w * c, pos[l.i], last[l.i]])
        for l in self.layers:                                      # placed producers live in their concat's store
            if l.i in place:
                cat, off = place[l.i]
                if cat in place:
                    raise NotImplementedError(f"YOLOv7: concat {cat} feeds another concat")
                s = owner[cat]
                stores[s][1] = min(stores[s][1], pos[l.i])
                stores[s][2] = max(stores[s][2], last[l.i])
                self.views[l.i] = View(s, off, shape[l.i][2], shape[l.i][0], shape[l.i][1])
        for i, s in owner.items():
            self.views[i] = View(s, 0, shape[i][2], shape[i][0], shape[i][1])
        self.ld = {s: 0 for s in range(len(stores))}
        for i, v in self.views.items():
            if v.off == 0 and i in owner:
                self.ld[v.store] = v.c
        # share buffers: a store reuses the smallest free block that fits (blocks free once their last reader has run)
        blocks: List[List[int]] = []                               # [size, free from position]
        self.store_block: List[int] = []
        for size, first, lst in stores:
            fit = [b for b in range(len(blocks)) if blocks[b][1] < first and blocks[b][0] >= size]
            if fit:
                b = min(fit, key=lambda b: blocks[b][0])
            else:
                blocks.append([size, 0])
                b = len(blocks) - 1
            blocks[b][1] = lst
            self.store_block.append(b)
        self.block_elems = [b[0] for b in blocks]
        # scratch: im2col rows and the temporaries inside DownC / SPPCSPC
        col = tmp = 0
        for l in self.layers:
            h, w, c = shape[l.f[0]] if l.f[0] >= 0 else (IN_H, IN_W, 3)
            for name, cv in l.convs.items():
                if cv.k == 3:
                    ho, wo = (h - 1) // cv.stride + 1, (w - 1) // cv.stride + 1
                    cin = 16 if cv.w.shape[1] == 12 else cv.w.shape[1]
                    col = max(col, ho * wo * 9 * cin)
            if l.type == "DownC":
                tmp = max(tmp, h * w * c)
            elif l.type == "SPPCSPC":
                c_ = l.convs["cv1"].w.shape[0]
                tmp = max(tmp, h * w * 4 * c_)
        self.col_elems, self.tmp_elems = col, tmp
        # detection rows: level k's map is the size of its input
        self.levels = []
        row0 = 0
        for k, j in enumerate(self.layers[-1].f):
            h, w, _ = shape[j]
            self.levels.append((j, h, w, row0))
            row0 += self.na * h * w
        self.R = row0
        assert self.R <= MAX_NMS, "more candidate rows than yolov7's max_nms"
        self.head_ld = (self.na * self.no + 7) // 8 * 8

    def peak_bytes(self, B: int) -> int:
        """Device bytes of activations, scratch and post-process buffers at batch B."""
        act = sum(self.block_elems) * 2 + (self.col_elems + 2 * self.tmp_elems) * 2
        head = sum(h * w for _, h, w, _ in self.levels) * self.head_ld * 2
        post = self.R * (8 * 4 + 4) + MAX_DET * (4 + 16 + 4 + 4) + 16
        return B * (act + head + post)

    # ------------------------------------------------------------------------------------------------------------ buffers
    def _buffers(self, B: int) -> dict:
        if B not in self._bufs:
            d = self.dev
            blk = [torch.empty(B * n, dtype=F16, device=d) for n in self.block_elems]
            bufs = {
                "blocks": blk,
                "col": torch.empty(max(B * self.col_elems, 8), dtype=F16, device=d),
                "tmp": [torch.empty(max(B * self.tmp_elems, 8), dtype=F16, device=d) for _ in range(2)],
                "head": [torch.empty(B * h * w * self.head_ld, dtype=F16, device=d) for _, h, w, _ in self.levels],
                "cand": torch.empty(B * self.R * 8, dtype=torch.float32, device=d),
                "count": torch.zeros(B, dtype=torch.int32, device=d),
                "order": torch.empty(B * self.R, dtype=torch.int32, device=d),
                "keep": torch.empty(B * MAX_DET, dtype=torch.int32, device=d),
                "nkeep": torch.empty(B, dtype=torch.int32, device=d),
                "boxes": torch.empty(B, MAX_DET, 4, dtype=torch.float32, device=d),
                "scores": torch.empty(B, MAX_DET, dtype=torch.float32, device=d),
                "classes": torch.empty(B, MAX_DET, dtype=torch.int32, device=d),
                "counts": torch.empty(B, dtype=torch.int32, device=d),
            }
            self._bufs[B] = bufs
        return self._bufs[B]

    def _rows(self, bufs, B: int, i: int) -> torch.Tensor:
        """Layer i's output as a [B*h*w, c] view with the store's row stride."""
        v = self.views[i]
        ld = self.ld[v.store]
        t = bufs["blocks"][self.store_block[v.store]][:B * v.h * v.w * ld].view(B * v.h * v.w, ld)
        return t[:, v.off:v.off + v.c]

    # ------------------------------------------------------------------------------------------------------------ launches
    def _conv(self, key, x: torch.Tensor, B: int, h: int, w: int, out: torch.Tensor, bufs, epi: int = _lib.EPI_BIAS_SILU_F16) -> None:
        """x [B*h*w, cin] rows (row stride allowed) -> out rows, conv `key` (1x1: GEMM; 3x3: im2col + GEMM)."""
        wt, b, k, s = self.w[key]
        if k == 1:
            gemm_f16(x, wt, b, epi, out=out)
            return
        ho, wo = (h - 1) // s + 1, (w - 1) // s + 1
        M, K = B * ho * wo, wt.shape[1]
        col = im2col(x, B, h, w, 3, s, bufs["col"][:M * K].view(M, K))
        gemm_f16(col, wt, b, epi, out=out)

    def _tmp(self, bufs, n: int, rows: int, c: int) -> torch.Tensor:
        return bufs["tmp"][n][:rows * c].view(rows, c)

    def _layer(self, l: Layer, bufs, B: int) -> None:
        st = _lib.stream_ptr()
        out = self._rows(bufs, B, l.i) if l.type not in ("Concat", "Detect") else None
        if l.type == "Conv":
            h, w, _ = self.shape[l.f[0]]
            self._conv((l.i, ""), self._rows(bufs, B, l.f[0]), B, h, w, out, bufs)
        elif l.type == "DownC":
            h, w, c = self.shape[l.f[0]]
            x = self._rows(bufs, B, l.f[0])
            c2 = l.convs["cv2"].w.shape[0]
            t = self._tmp(bufs, 0, B * h * w, c)
            self._conv((l.i, "cv1"), x, B, h, w, t, bufs)
            self._conv((l.i, "cv2"), t, B, h, w, out[:, :c2], bufs)
            p = self._tmp(bufs, 1, B * (h // 2) * (w // 2), c)
            _lib.check(self.lib.vlfm_yolo_maxpool2(x.data_ptr(), x.stride(0), p.data_ptr(), c, B, h, w, c, st), "vlfm_yolo_maxpool2")
            self._conv((l.i, "cv3"), p, B, h // 2, w // 2, out[:, c2:], bufs)
        elif l.type == "SPPCSPC":
            h, w, _ = self.shape[l.f[0]]
            x = self._rows(bufs, B, l.f[0])
            c_ = l.convs["cv1"].w.shape[0]
            rows = B * h * w
            cat4 = self._tmp(bufs, 0, rows, 4 * c_)
            t1 = self._tmp(bufs, 1, rows, c_)
            self._conv((l.i, "cv1"), x, B, h, w, t1, bufs)
            t2 = bufs["tmp"][1][rows * c_:2 * rows * c_].view(rows, c_)
            self._conv((l.i, "cv3"), t1, B, h, w, t2, bufs)
            self._conv((l.i, "cv4"), t2, B, h, w, cat4[:, :c_], bufs)
            _lib.check(self.lib.vlfm_yolo_spp_pools(cat4.data_ptr(), 4 * c_, cat4[:, c_:].data_ptr(), 4 * c_, B, h, w, c_, st),
                       "vlfm_yolo_spp_pools")
            t3 = self._tmp(bufs, 1, rows, c_)
            self._conv((l.i, "cv5"), cat4, B, h, w, t3, bufs)
            cat2 = self._tmp(bufs, 0, rows, 2 * c_)
            self._conv((l.i, "cv6"), t3, B, h, w, cat2[:, :c_], bufs)
            self._conv((l.i, "cv2"), x, B, h, w, cat2[:, c_:], bufs)
            self._conv((l.i, "cv7"), cat2, B, h, w, out, bufs)
        elif l.type == "Upsample":
            h, w, c = self.shape[l.f[0]]
            x = self._rows(bufs, B, l.f[0])
            _lib.check(self.lib.vlfm_yolo_upsample2(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), B, h, w, c, st),
                       "vlfm_yolo_upsample2")
        elif l.type == "Shortcut":
            a, b = self._rows(bufs, B, l.f[0]), self._rows(bufs, B, l.f[1])
            _lib.check(self.lib.vlfm_yolo_add(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
                                              a.shape[0], a.shape[1], st), "vlfm_yolo_add")
        elif l.type == "Detect":
            for k, (j, h, w, _) in enumerate(self.levels):
                head = bufs["head"][k].view(B * h * w, self.head_ld)[:, :self.na * self.no]
                self._conv((l.i, f"m{k}"), self._rows(bufs, B, j), B, h, w, head, bufs, epi=_lib.EPI_BIAS_F16)
        # ReOrg is written by the preprocess launch; Concat's inputs already sit in its buffer

    def _forward(self, images: torch.Tensor, B: int, H: int, W: int, bufs) -> None:
        st = _lib.stream_ptr()
        yo, ys, yb, xo, xs, xa = self._tables[(H, W)]
        x0 = self._rows(bufs, B, self.layers[0].i)
        _lib.check(self.lib.vlfm_yolo_preprocess(images.data_ptr(), x0.data_ptr(), B, H, W, IN_H, IN_W, yo.data_ptr(), ys.data_ptr(),
                                                 yb.data_ptr(), xo.data_ptr(), xs.data_ptr(), xa.data_ptr(), st), "vlfm_yolo_preprocess")
        for l in self.layers[1:]:
            self._layer(l, bufs, B)
        self.postprocess(B, H, W, bufs)

    def postprocess(self, B: int, H: int, W: int, bufs) -> None:
        """Decode the head tensors in bufs["head"], sort, NMS and map the boxes into bufs["boxes" / "scores" / "classes" / "counts"]."""
        st = _lib.stream_ptr()
        bufs["count"].zero_()
        for k, (_, h, w, row0) in enumerate(self.levels):
            _lib.check(self.lib.vlfm_yolo_decode(bufs["head"][k].data_ptr(), self.head_ld, B, h, w, self.na, self.nc,
                                                 self.anchors[k].data_ptr(), self.strides[k], row0, self.R, self.params.data_ptr(),
                                                 bufs["cand"].data_ptr(), bufs["count"].data_ptr(), st), "vlfm_yolo_decode")
        _lib.check(self.lib.vlfm_yolo_sort(bufs["cand"].data_ptr(), bufs["count"].data_ptr(), self.R, B, bufs["order"].data_ptr(), st),
                   "vlfm_yolo_sort")
        _lib.check(self.lib.vlfm_yolo_nms(bufs["cand"].data_ptr(), bufs["order"].data_ptr(), bufs["count"].data_ptr(), self.R, B,
                                          self.params.data_ptr(), MAX_DET, bufs["keep"].data_ptr(), bufs["nkeep"].data_ptr(), st),
                   "vlfm_yolo_nms")
        gain, px, py = scale_coords_params(H, W)
        _lib.check(self.lib.vlfm_yolo_boxes(bufs["cand"].data_ptr(), bufs["keep"].data_ptr(), bufs["nkeep"].data_ptr(), self.R, B, MAX_DET,
                                            gain, px, py, H, W, bufs["boxes"].data_ptr(), bufs["scores"].data_ptr(),
                                            bufs["classes"].data_ptr(), bufs["counts"].data_ptr(), st), "vlfm_yolo_boxes")

    # -------------------------------------------------------------------------------------------------------------- API
    def set_params(self, conf_thres: float, iou_thres: float, classes: Optional[Sequence[int]], agnostic: bool) -> None:
        p = _lib.YoloParams()
        p.conf_thres, p.iou_thres, p.agnostic = float(conf_thres), float(iou_thres), int(bool(agnostic))
        mask = [0, 0, 0, 0]
        for j in (range(self.nc) if classes is None else classes):
            if not 0 <= int(j) < self.nc:
                continue                      # yolov7 compares class indices: an absent index keeps nothing
            mask[int(j) >> 5] |= 1 << (int(j) & 31)
        for k in range(4):
            p.class_mask[k] = mask[k]
        host = torch.frombuffer(bytearray(C.string_at(C.addressof(p), C.sizeof(p))), dtype=torch.int32)
        self.params.copy_(host)

    def _prepare(self, H: int, W: int) -> None:
        if (H, W) not in self._tables:
            yo, ys, yb = area_tables(H, IN_H)
            xo, xs, xa = area_tables(W, IN_W)
            self._tables[(H, W)] = tuple(torch.from_numpy(a).to(self.dev) for a in (yo, ys, yb, xo, xs, xa))

    @torch.inference_mode()
    def run(self, images: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """images [B,H,W,3] uint8 RGB (device) -> views of (boxes [B,300,4], scores [B,300], classes [B,300], counts [B]); valid
        until the next call with the same B."""
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3:
            raise ValueError(f"YOLOv7: expected uint8 frames [B, H, W, 3], got {tuple(images.shape)} {images.dtype}")
        B, H, W = images.shape[:3]
        check_frame(H, W)
        with torch.cuda.device(self.dev):
            self._prepare(H, W)
            bufs = self._buffers(B)
            self.graphs((B, H, W), self.use_graph, lambda x: self._forward(x, B, H, W, bufs), images.contiguous())
        return bufs["boxes"], bufs["scores"], bufs["classes"], bufs["counts"]
