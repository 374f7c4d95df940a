"""Detection path: host-side mirror of `DetectionPredictor.model` over the CUDA detection engine.

  * pack_det_program   reference-named state dict -> (op program, packed weights): BatchNorm folded in fp32,
                       NHWC / K-major weight layouts, buffer plan
  * DetEngine          ctypes wrapper of sb_det_* (include/surya_b200.h)
  * B200EfficientViT   quacks like EfficientViTForSemanticSegmentation for the predictor
                       (surya/detection/__init__.py:70, 111-120): model(pixel_values=...) -> .logits, .config.num_labels,
                       .dtype, .device
  * detect_heatmaps    the predictor's model call + x4 bilinear upsample + .float() (:115-132) on the device

No PyTorch math on the forward path and no import of oracle/.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Dict, List, Tuple

import torch

from . import _lib
from ._lib import c_int, c_void_p, check, ptr, stream_ptr
from .config import DetConfig
from .det_arch import Block, ConvSpec, det_blocks, det_head_specs
from .ops import ACT, dt_code

OP_STEM, OP_CONV, OP_PW, OP_DW, OP_GPW, OP_MLA, OP_UPCAT, OP_CLS = range(8)

# Capacity of sb_det_text_boxes' per-page tables: text lines, and points (two per dilated row of each line).  A page beyond
# either goes through the host path.
DEFAULT_MAX_BOXES = 1024
DEFAULT_MAX_POINTS = 65536


def box_tables(n: int, max_boxes: int, max_points: int, device=None) -> Dict[str, torch.Tensor]:
    """Output tables of sb_det_text_boxes for n pages (include/surya_b200.h); pinned host tensors when device is None."""
    t = {"count": torch.empty((n,), dtype=torch.int32, device=device),
         "overflow": torch.empty((n,), dtype=torch.int32, device=device),
         "box": torch.empty((n, max_boxes, 7), dtype=torch.int32, device=device),
         "peak": torch.empty((n, max_boxes), dtype=torch.float32, device=device),
         "points": torch.empty((n, max_points, 2), dtype=torch.int32, device=device)}
    return t if device is not None else {k: v.pin_memory() for k, v in t.items()}


class _DetOpC(ctypes.Structure):
    _fields_ = [
        ("op", c_int), ("src", c_int * 4), ("n_src", c_int), ("src_off", c_int * 4), ("dst", c_int), ("res", c_int),
        ("w", c_int), ("b", c_int), ("cin", c_int), ("cout", c_int), ("k", c_int), ("stride", c_int), ("pad", c_int),
        ("act", c_int), ("groups", c_int), ("heads", c_int), ("dim", c_int), ("eps", ctypes.c_float),
    ]


@dataclass
class DetProgram:
    ops: List[dict]
    weights: List[torch.Tensor]
    n_bufs: int
    buf_names: List[str]


def _fold(sd: Dict[str, torch.Tensor], c: ConvSpec) -> Tuple[torch.Tensor, torch.Tensor | None]:
    """Conv weight/bias with the following BatchNorm2d(eval) folded in, fp32 (ConvNormAct: encoderdecoder.py:82-86)."""
    w = sd[c.wkey].float()
    b = sd[c.bkey].float() if c.bias else None
    if c.norm:
        n = f"{c.name}.norm"
        scale = sd[f"{n}.weight"].float() / torch.sqrt(sd[f"{n}.running_var"].float() + c.eps)
        shift = sd[f"{n}.bias"].float() - sd[f"{n}.running_mean"].float() * scale
        w = w * scale.view(-1, 1, 1, 1)
        b = shift if b is None else b * scale + shift
    return w, b


def pack_det_program(sd: Dict[str, torch.Tensor], cfg: DetConfig, dtype: torch.dtype, device) -> DetProgram:
    weights: List[torch.Tensor] = []
    ops: List[dict] = []
    names: List[str] = []

    def buf(name: str) -> int:
        names.append(name)
        return len(names) - 1

    def W(t: torch.Tensor, keep_f32: bool = False) -> int:
        weights.append((t.float() if keep_f32 else t.to(dtype)).contiguous().to(device))
        return len(weights) - 1

    def emit(op, src, dst, res=-1, w=-1, b=-1, cin=0, cout=0, k=1, stride=1, pad=0, act="none", groups=1, heads=0, dim=0,
             eps=0.0, src_off=(0, 0, 0, 0)):
        src = list(src) + [-1] * (4 - len(src))
        ops.append(dict(op=op, src=src, n_src=sum(1 for s in src if s != -1), src_off=list(src_off), dst=dst, res=res, w=w, b=b,
                        cin=cin, cout=cout, k=k, stride=stride, pad=pad, act=ACT[act], groups=groups, heads=heads, dim=dim,
                        eps=eps))

    def conv_op(c: ConvSpec, src: int, dst: int, res: int = -1):
        w, b = _fold(sd, c)
        bi = W(b, keep_f32=True) if b is not None else -1
        if c.groups == 1 and c.k == 1:
            emit(OP_PW, [src], dst, res, W(w.reshape(c.cout, c.cin)), bi, c.cin, c.cout, act=c.act)
        elif c.groups == 1:
            emit(OP_CONV, [src], dst, res, W(w.permute(0, 2, 3, 1).reshape(c.cout, -1)), bi, c.cin, c.cout, c.k, c.stride,
                 c.pad if not c.bare else c.k // 2, c.act)
        elif c.groups == c.cin:
            emit(OP_DW, [src], dst, res, W(w.reshape(c.cout, c.k * c.k).t()), bi, c.cin, c.cout, c.k, c.stride,
                 c.pad if not c.bare else c.k // 2, c.act, groups=c.groups)
        else:
            gk = c.cin // c.groups
            wp = torch.zeros((c.cout, 64), dtype=torch.float32)
            wp[:, :gk] = w.reshape(c.cout, gk)
            assert b is None
            emit(OP_GPW, [src], dst, res, W(wp), -1, c.cin, c.cout, groups=c.groups)

    X = [buf("x0"), buf("x1")]
    T1, T2 = buf("t1"), buf("t2")
    Q1, Q2, Q3, M = buf("mla_qkv"), buf("mla_dw"), buf("mla_agg"), buf("mla_out")
    n_stage = len(cfg.widths) - 1
    F = [buf(f"feat{i}") for i in range(n_stage)]
    blocks = det_blocks(cfg)
    last_of_stage = {}
    for i, blk in enumerate(blocks):
        if blk.stage >= 0:
            last_of_stage[blk.stage] = i
    cur = -2
    for i, blk in enumerate(blocks):
        is_last = blk.stage >= 0 and last_of_stage[blk.stage] == i

        def other(c):
            return X[1] if c == X[0] else X[0]

        out = F[blk.stage] if is_last else other(cur)
        if blk.kind == "conv":      # stem in_conv, reads the NCHW pixel batch
            c = blk.convs[0]
            w, b = _fold(sd, c)
            emit(OP_STEM, [-2], out, -1, W(w.permute(0, 2, 3, 1).reshape(c.cout, -1), True), W(b, True), c.cin, c.cout, c.k,
                 c.stride, c.pad, c.act)
        elif blk.kind in ("convblock", "fused"):
            conv_op(blk.convs[0], cur, T1)
            conv_op(blk.convs[1], T1, out, cur if blk.residual else -1)
        elif blk.kind == "mb":
            conv_op(blk.convs[0], cur, T1)
            conv_op(blk.convs[1], T1, T2)
            conv_op(blk.convs[2], T2, out, cur if blk.residual else -1)
        elif blk.kind == "vit":
            qkv_c, dw_c, pw_c, proj_c = blk.mla
            conv_op(qkv_c, cur, Q1)
            conv_op(dw_c, Q1, Q2)
            conv_op(pw_c, Q2, Q3)
            emit(OP_MLA, [Q1, Q3], M, heads=blk.heads, dim=blk.dim, eps=cfg.mla_eps, cin=3 * blk.heads * blk.dim,
                 cout=2 * blk.heads * blk.dim)
            mid = other(cur)
            conv_op(proj_c, M, mid, cur)                 # context module + identity shortcut
            final = F[blk.stage] if is_last else cur     # `cur` is dead once the context module is done
            conv_op(blk.convs[0], mid, T1)
            conv_op(blk.convs[1], T1, T2)
            conv_op(blk.convs[2], T2, final, mid)        # local module + identity shortcut
            out = final
        else:
            raise ValueError(blk.kind)
        cur = out

    # ---- decode head (encoderdecoder.py:699-722)
    hs = det_head_specs(cfg)
    dl = cfg.decoder_layer_hidden_size
    P = [buf(f"proj{i}") for i in range(n_stage)]
    for i, (name, cin, cout) in enumerate(hs["linear_c"]):
        emit(OP_PW, [F[i]], P[i], -1, W(sd[f"{name}.weight"]), W(sd[f"{name}.bias"].to(dtype), True), cin, cout)
    CAT, FUSED = buf("cat"), buf("fused")
    offs = [(n_stage - 1 - i) * dl for i in range(n_stage)]      # torch.cat(all_hidden_states[::-1])
    emit(OP_UPCAT, P, CAT, cin=dl, cout=dl * n_stage, src_off=offs)
    name, cin, cout = hs["fuse"]
    bn = hs["bn"]
    scale = sd[f"{bn}.weight"].float() / torch.sqrt(sd[f"{bn}.running_var"].float() + cfg.head_bn_eps)
    shift = sd[f"{bn}.bias"].float() - sd[f"{bn}.running_mean"].float() * scale
    emit(OP_PW, [CAT], FUSED, -1, W(sd[f"{name}.weight"].float().reshape(cout, cin) * scale.view(-1, 1)), W(shift, True), cin,
         cout, act="relu")
    name, cin, cout = hs["cls"]
    emit(OP_CLS, [FUSED], -3, -1, W(sd[f"{name}.weight"].reshape(cout, cin)), W(sd[f"{name}.bias"]), cin, cout)
    return DetProgram(ops=ops, weights=weights, n_bufs=len(names), buf_names=names)


def plan_buffers(prog: DetProgram, H: int, W: int) -> List[int]:
    """Per-image element capacity of every workspace buffer for an H x W input (shape simulation of the program)."""
    dims: Dict[int, Tuple[int, int, int]] = {}
    cap = [0] * prog.n_bufs
    for op in prog.ops:
        s0 = op["src"][0]
        h, w = (H, W) if s0 < 0 else dims[s0][:2]
        if op["op"] == OP_STEM:
            od = (H // 2, W // 2, op["cout"])
        elif op["op"] in (OP_CONV, OP_DW):
            od = ((h + 2 * op["pad"] - op["k"]) // op["stride"] + 1, (w + 2 * op["pad"] - op["k"]) // op["stride"] + 1, op["cout"])
        else:
            od = (h, w, op["cout"])
        if op["dst"] >= 0:
            dims[op["dst"]] = od
            cap[op["dst"]] = max(cap[op["dst"]], od[0] * od[1] * od[2])
    return cap


class DetEngine:
    def __init__(self, cfg: DetConfig, state_dict: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float16,
                 device: str | torch.device = "cuda", max_batch: int = 8, max_hw: Tuple[int, int] = (1024, 1024)):
        self.lib = _lib.load()
        self.cfg, self.dtype, self.device = cfg, dtype, torch.device(device)
        self.prog = pack_det_program(state_dict, cfg, dtype, self.device)
        self.max_batch, self.max_hw = max_batch, max_hw
        caps = plan_buffers(self.prog, *max_hw)
        n = len(self.prog.ops)
        arr = (_DetOpC * n)()
        for i, o in enumerate(self.prog.ops):
            c = arr[i]
            c.op, c.n_src, c.dst, c.res, c.w, c.b = o["op"], o["n_src"], o["dst"], o["res"], o["w"], o["b"]
            for j in range(4):
                c.src[j] = o["src"][j]
                c.src_off[j] = o["src_off"][j]
            c.cin, c.cout, c.k, c.stride, c.pad, c.act, c.groups = o["cin"], o["cout"], o["k"], o["stride"], o["pad"], o["act"], o["groups"]
            c.heads, c.dim, c.eps = o["heads"], o["dim"], o["eps"]
        wptr = (c_void_p * len(self.prog.weights))(*[w.data_ptr() for w in self.prog.weights])
        caps_c = (ctypes.c_longlong * len(caps))(*caps)
        self._h = c_void_p()
        self.lib.sb_det_workspace_bytes.restype = ctypes.c_size_t
        with torch.cuda.device(self.device):
            check(self.lib.sb_det_create(c_int(dt_code(dtype)), arr, c_int(n), wptr, c_int(len(self.prog.weights)), caps_c,
                                         c_int(len(caps)), c_int(max_batch), ctypes.byref(self._h)), "sb_det_create")

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.sb_det_destroy(self._h)
            self._h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def workspace_bytes(self) -> int:
        return int(self.lib.sb_det_workspace_bytes(self._h))

    def forward(self, pixel_values: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """pixel_values NCHW [B,3,H,W] on the device (fp32 or engine dtype) -> sigmoid maps [B, num_labels, H/4, W/4]."""
        B, C, H, W = pixel_values.shape
        if not pixel_values.is_cuda:
            pixel_values = pixel_values.to(self.device, non_blocking=True)
        pixel_values = pixel_values.contiguous()
        f32 = pixel_values.dtype == torch.float32
        if not f32 and pixel_values.dtype != self.dtype:
            raise _lib.SuryaB200Error(f"pixel_values must be float32 or {self.dtype}")
        if H > self.max_hw[0] or W > self.max_hw[1] or H % 32 or W % 32:
            raise _lib.SuryaB200Error(f"input {H}x{W} must be a multiple of 32 and within {self.max_hw}")
        if out is None:
            out = torch.empty((B, self.cfg.num_labels, H // 4, W // 4), dtype=self.dtype, device=self.device)
        for b0 in range(0, B, self.max_batch):
            b1 = min(B, b0 + self.max_batch)
            check(self.lib.sb_det_forward(self._h, ptr(pixel_values[b0:b1]), c_int(1 if f32 else 0), c_int(b1 - b0), c_int(H),
                                          c_int(W), ptr(out[b0:b1]), stream_ptr()), "sb_det_forward")
        return out

    def upsample(self, logits: torch.Tensor, size: Tuple[int, int], out: torch.Tensor | None = None) -> torch.Tensor:
        """F.interpolate(logits, size, mode='bilinear', align_corners=False).float() (surya/detection/__init__.py:120-132)."""
        B, L, hs, ws = logits.shape
        if out is None:
            out = torch.empty((B, L, size[0], size[1]), dtype=torch.float32, device=logits.device)
        check(self.lib.sb_det_upsample(c_int(dt_code(logits.dtype)), ptr(logits.contiguous()), ptr(out), c_int(B * L), c_int(hs),
                                       c_int(ws), c_int(size[0]), c_int(size[1]), stream_ptr()), "sb_det_upsample")
        return out

    def normalize_u8(self, pages: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """uint8 NHWC [B,H,W,3] device tensor -> normalised NCHW [B,3,H,W] in the engine dtype (sb_det_normalize_u8)."""
        B, H, W, C = pages.shape
        assert C == 3 and pages.dtype == torch.uint8 and pages.is_cuda
        if out is None:
            out = torch.empty((B, 3, H, W), dtype=self.dtype, device=pages.device)
        check(self.lib.sb_det_normalize_u8(c_int(dt_code(self.dtype)), ptr(pages.contiguous()), ptr(out), c_int(B), c_int(H),
                                           c_int(W), stream_ptr()), "sb_det_normalize_u8")
        return out

    def text_front(self, logits: torch.Tensor, size: Tuple[int, int], text_threshold: float = 0.6, low_text: float = 0.35,
                   out: Dict[str, torch.Tensor] | None = None) -> Dict[str, torch.Tensor]:
        """Device-side front half of the detection post-processing for the TEXT channel (sb_det_text_front): the x4 bilinear map
        in the engine dtype (exactly the values `F.interpolate(...).to(float32)` holds, surya/detection/__init__.py:120-132), the
        dynamic thresholds of get_dynamic_thresholds (surya/detection/heatmap.py:14-24; defaults = settings.DETECTOR_TEXT_THRESHOLD
        / DETECTOR_BLANK_THRESHOLD) and the binarised `map > low_text` mask (:33).  Returns device tensors
        {"map": [B,H,W] dtype, "mask": [B,H,W] uint8, "thr": [B,4] fp32 (text_threshold, low_text, top-10 % mean, scale)}."""
        B, L, hs, ws = logits.shape
        H, W = size
        dev = logits.device
        if out is None:
            out = {"map": torch.empty((B, H, W), dtype=logits.dtype, device=dev),
                   "mask": torch.empty((B, H, W), dtype=torch.uint8, device=dev),
                   "thr": torch.empty((B, 4), dtype=torch.float32, device=dev)}
        hist = getattr(self, "_front_hist", None)
        if hist is None or hist.shape[0] < B:
            hist = torch.zeros((max(B, self.max_batch), 16384), dtype=torch.int32, device=dev)
            self._front_hist = hist
        check(self.lib.sb_det_text_front(c_int(dt_code(logits.dtype)), ptr(logits.contiguous()), c_int(L), c_int(B), c_int(hs),
                                         c_int(ws), c_int(H), c_int(W), ptr(out["map"]), ptr(out["mask"]), ptr(out["thr"]),
                                         ptr(hist), ctypes.c_float(text_threshold), ctypes.c_float(low_text), stream_ptr()),
              "sb_det_text_front")
        return out

    def text_boxes(self, front: Dict[str, torch.Tensor], max_boxes: int = DEFAULT_MAX_BOXES, max_points: int = DEFAULT_MAX_POINTS,
                   out: Dict[str, torch.Tensor] | None = None) -> Dict[str, torch.Tensor]:
        """Back half of detect_boxes (surya/detection/heatmap.py:33-107) on the device (sb_det_text_boxes) for text_front()'s
        output: connected components, size / peak filter and the dilated row extents as per-page device tables
        {"count": [B], "overflow": [B], "box": [B, max_boxes, 7] (dilated x0, y0, x1, y1, point offset, point count, ks),
        "peak": [B, max_boxes], "points": [B, max_points, 2]}.  text_boxes_from_tables() finishes one page on the host."""
        front = {k: front[k].contiguous() for k in ("map", "mask", "thr")}
        B, H, W = front["map"].shape
        dev = front["map"].device
        if out is None:
            out = box_tables(B, max_boxes, max_points, device=dev)
        need = B * (18 * H * W + 8 * H + 4 * max_points + 20)
        scratch = getattr(self, "_boxes_scratch", None)
        if scratch is None or scratch.numel() < need:
            scratch = torch.empty((need,), dtype=torch.uint8, device=dev)
            self._boxes_scratch = scratch
        check(self.lib.sb_det_text_boxes(c_int(dt_code(front["map"].dtype)), ptr(front["map"]), ptr(front["mask"]), ptr(front["thr"]),
                                         c_int(B), c_int(H), c_int(W), c_int(max_boxes), c_int(max_points), ptr(scratch),
                                         ctypes.c_size_t(scratch.numel()), ptr(out["count"]), ptr(out["overflow"]), ptr(out["box"]),
                                         ptr(out["peak"]), ptr(out["points"]), stream_ptr()), "sb_det_text_boxes")
        return out

    def page_resize(self, pages_dev: torch.Tensor, plan, processor_size: Tuple[int, int], out: torch.Tensor | None = None) -> torch.Tensor:
        """sb_det_page_resize: the packed uint8 pages of `plan` (a page_prep.PagePlan) on the device -> processor-size uint8 chunks
        [n_chunks, H, W, 3], byte-equal to split_image + prepare_image's PIL chain.  processor_size = (width, height)."""
        pw, ph = processor_size
        dev = pages_dev.device
        n = len(plan.chunks)
        if out is None:
            out = torch.empty((n, ph, pw, 3), dtype=torch.uint8, device=dev)
        scratch = getattr(self, "_resize_scratch", None)
        if plan.scratch_bytes and (scratch is None or scratch.numel() < plan.scratch_bytes):
            scratch = torch.empty((plan.scratch_bytes,), dtype=torch.uint8, device=dev)
            self._resize_scratch = scratch
        desc = torch.from_numpy(plan.desc).to(dev, non_blocking=True)
        tables = torch.from_numpy(plan.tables).to(dev, non_blocking=True)
        steps = len(plan.step_jobs)
        check(self.lib.sb_det_page_resize(ptr(pages_dev), ptr(scratch if plan.scratch_bytes else None), ptr(out), ptr(desc),
                                          ptr(tables), c_int(steps), (c_int * steps)(*plan.step_jobs),
                                          (ctypes.c_longlong * steps)(*plan.step_max_px), stream_ptr()), "sb_det_page_resize")
        return out

    def text_front_stitched(self, logits: torch.Tensor, plan, size: Tuple[int, int], text_threshold: float = 0.6,
                            low_text: float = 0.35) -> Dict[str, torch.Tensor]:
        """text_front over the chunks of `plan`, stitched per page (sb_det_text_front_stitched): {"map": [rows, W] packed over
        the pages (page p at rows plan.page_tab[p, 0] ...), "mask": same, "thr": [n_pages, 4]}.  size = (H, W) of a chunk."""
        n, L, hs, ws = logits.shape
        H, W = size
        dev = logits.device
        P = plan.page_tab.shape[0]
        rows = int(plan.page_tab[:, 1].sum())
        out = {"map": torch.empty((rows, W), dtype=logits.dtype, device=dev), "mask": torch.empty((rows, W), dtype=torch.uint8, device=dev),
               "thr": torch.empty((P, 4), dtype=torch.float32, device=dev)}
        hist = getattr(self, "_front_hist", None)
        if hist is None or hist.shape[0] < P:
            hist = torch.zeros((max(P, self.max_batch), 16384), dtype=torch.int32, device=dev)
            self._front_hist = hist
        chunk_tab = torch.from_numpy(plan.chunk_tab).to(dev, non_blocking=True)
        page_tab = torch.from_numpy(plan.page_tab).to(dev, non_blocking=True)
        check(self.lib.sb_det_text_front_stitched(c_int(dt_code(logits.dtype)), ptr(logits.contiguous()), c_int(L), c_int(n), c_int(hs),
                                                  c_int(ws), c_int(H), c_int(W), ptr(chunk_tab), c_int(P), ptr(page_tab),
                                                  c_int(int(plan.page_tab[:, 1].max())), ptr(out["map"]), ptr(out["mask"]),
                                                  ptr(out["thr"]), ptr(hist), ctypes.c_float(text_threshold),
                                                  ctypes.c_float(low_text), stream_ptr()), "sb_det_text_front_stitched")
        return out

    def debug_buffer(self, name: str, B: int, H: int, W: int, C: int) -> torch.Tensor:
        idx = self.prog.buf_names.index(name)
        out = torch.empty((B, H, W, C), dtype=self.dtype, device=self.device)
        check(self.lib.sb_det_debug_copy(self._h, c_int(idx), ptr(out), ctypes.c_size_t(out.numel() * 2), stream_ptr()),
              "sb_det_debug_copy")
        return out


class _Out:
    def __init__(self, logits):
        self.logits = logits


class _DetCfg:
    def __init__(self, cfg: DetConfig):
        self.__dict__.update(cfg.to_dict())


class B200EfficientViT:
    """Call-compatible with what DetectionPredictor touches on `self.model`
    (surya/detection/__init__.py:70 config.num_labels, :111-118 model(pixel_values=...).logits, .dtype, .device)."""

    def __init__(self, engine: DetEngine):
        self.engine = engine
        self.config = _DetCfg(engine.cfg)
        self.device, self.dtype = engine.device, engine.dtype

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def __call__(self, pixel_values: torch.Tensor):
        return _Out(self.engine.forward(pixel_values))


def detect_heatmaps(engine: DetEngine, pixel_values: torch.Tensor, out_size: Tuple[int, int] | None = None) -> torch.Tensor:
    """DetectionPredictor.batch_detection's device part (surya/detection/__init__.py:115-132): forward, bilinear upsample
    to the processor size, float32.  Returns a device tensor [B, 2, H, W] (caller does the D2H copy)."""
    logits = engine.forward(pixel_values)
    size = out_size or tuple(pixel_values.shape[2:])
    return engine.upsample(logits, size)


def detect_pages_host(engine: DetEngine, pages_host: torch.Tensor, out_host: torch.Tensor | None = None, chunk: int = 8,
                      out_size: Tuple[int, int] | None = None, sync: bool = True) -> torch.Tensor:
    """Host-to-host variant of detect_heatmaps for a whole batch (DetectionPredictor.batch_detection,
    surya/detection/__init__.py:94-132: pixel batch up, fp32 full-resolution heatmaps down): the batch is cut into chunks and
    the upload of chunk i+1, the forward + upsample of chunk i and the download of chunk i-1 run on three streams, so PCIe
    time hides behind the kernels.  pages_host: pinned NCHW fp16/fp32 [B,3,H,W]; returns pinned fp32 [B, labels, H, W], complete
    on return (sync=False returns after stream-ordering only: the caller must synchronise before touching the buffer)."""
    B, _, H, W = pages_host.shape
    size = out_size or (H, W)
    L = engine.cfg.num_labels
    dev = engine.device
    if out_host is None:
        out_host = torch.empty((B, L, size[0], size[1]), dtype=torch.float32).pin_memory()
    st = getattr(engine, "_pipe", None)
    key = (chunk, H, W, size, pages_host.dtype)
    if st is None or st["key"] != key:
        st = {"key": key, "s_in": torch.cuda.Stream(dev), "s_c": torch.cuda.Stream(dev), "s_out": torch.cuda.Stream(dev),
              "x": [torch.empty((chunk, 3, H, W), dtype=pages_host.dtype, device=dev) for _ in range(2)],
              "up": [torch.empty((chunk, L, size[0], size[1]), dtype=torch.float32, device=dev) for _ in range(2)],
              "lg": [torch.empty((chunk, L, H // 4, W // 4), dtype=engine.dtype, device=dev) for _ in range(2)]}
        engine._pipe = st
    s_in, s_c, s_out = st["s_in"], st["s_c"], st["s_out"]
    cur = torch.cuda.current_stream(dev)
    for s_ in (s_in, s_c, s_out):
        s_.wait_stream(cur)
    ev_c = [None, None]      # compute finished on buffer k  (guards re-upload into x[k])
    ev_o = [None, None]      # download finished on buffer k (guards re-use of up[k])
    for i, b0 in enumerate(range(0, B, chunk)):
        b1 = min(B, b0 + chunk)
        n, k = b1 - b0, i & 1
        with torch.cuda.stream(s_in):
            if ev_c[k] is not None:
                s_in.wait_event(ev_c[k])
            st["x"][k][:n].copy_(pages_host[b0:b1], non_blocking=True)
            ev_in = torch.cuda.Event()
            ev_in.record(s_in)
        with torch.cuda.stream(s_c):
            s_c.wait_event(ev_in)
            if ev_o[k] is not None:
                s_c.wait_event(ev_o[k])
            engine.forward(st["x"][k][:n], out=st["lg"][k][:n])
            engine.upsample(st["lg"][k][:n], size, out=st["up"][k][:n])
            ev_c[k] = torch.cuda.Event()
            ev_c[k].record(s_c)
        with torch.cuda.stream(s_out):
            s_out.wait_event(ev_c[k])
            out_host[b0:b1].copy_(st["up"][k][:n], non_blocking=True)
            ev_o[k] = torch.cuda.Event()
            ev_o[k].record(s_out)
    cur.wait_stream(s_out)
    cur.wait_stream(s_c)
    if sync:
        # host-to-host contract: the caller reads out_host (e.g. `.numpy()`, like the reference after `.cpu()`) right away,
        # so the last download must have landed, not merely be ordered on a stream
        for ev in ev_o:
            if ev is not None:
                ev.synchronize()
    return out_host


def _front_pipeline(engine: DetEngine, pages_host: torch.Tensor, chunk: int, out_size: Tuple[int, int] | None,
                    text_threshold: float, low_text: float, sync: bool, tables: Tuple[int, int] | None = None):
    """Three-stream chunk pipeline of detect_text_front_host / detect_text_boxes_host: the upload of chunk i+1, normalise +
    forward + sb_det_text_front of chunk i and the download of chunk i-1 run on three streams, so PCIe time hides behind the
    kernels.  tables=None downloads the text front (map, mask, thresholds); tables=(max_boxes, max_points) runs
    sb_det_text_boxes after the front and downloads only its tables.  Returns pinned tensors indexed by page."""
    u8 = pages_host.dtype == torch.uint8        # raw pages [B,H,W,3]: normalised on the device (3 bytes per pixel over PCIe)
    if u8:
        B, H, W, _ = pages_host.shape
    else:
        B, _, H, W = pages_host.shape
    size = out_size or (H, W)
    dev = engine.device
    L = engine.cfg.num_labels
    key = (chunk, H, W, size, pages_host.dtype, B, tables)
    attr = "_pipe_front" if tables is None else "_pipe_boxes"
    st = getattr(engine, attr, None)
    if st is None or st["key"] != key:
        front = [{"map": torch.empty((chunk, size[0], size[1]), dtype=engine.dtype, device=dev),
                  "mask": torch.empty((chunk, size[0], size[1]), dtype=torch.uint8, device=dev),
                  "thr": torch.empty((chunk, 4), dtype=torch.float32, device=dev)} for _ in range(2)]
        if tables is None:
            down = front
            host = {k: torch.empty((B,) + v.shape[1:], dtype=v.dtype).pin_memory() for k, v in front[0].items()}
        else:
            down = [box_tables(chunk, *tables, device=dev) for _ in range(2)]
            host = box_tables(B, *tables)
        st = {"key": key, "s_in": torch.cuda.Stream(dev), "s_c": torch.cuda.Stream(dev), "s_out": torch.cuda.Stream(dev),
              "x": [torch.empty((chunk, H, W, 3) if u8 else (chunk, 3, H, W), dtype=pages_host.dtype, device=dev) for _ in range(2)],
              "xn": [torch.empty((chunk, 3, H, W), dtype=engine.dtype, device=dev) for _ in range(2)] if u8 else None,
              "lg": [torch.empty((chunk, L, H // 4, W // 4), dtype=engine.dtype, device=dev) for _ in range(2)],
              "front": front, "down": down, "host": host}
        setattr(engine, attr, st)
    s_in, s_c, s_out = st["s_in"], st["s_c"], st["s_out"]
    host = st["host"]
    cur = torch.cuda.current_stream(dev)
    for s_ in (s_in, s_c, s_out):
        s_.wait_stream(cur)
    ev_c, ev_o = [None, None], [None, None]
    for i, b0 in enumerate(range(0, B, chunk)):
        b1 = min(B, b0 + chunk)
        n, k = b1 - b0, i & 1
        with torch.cuda.stream(s_in):
            if ev_c[k] is not None:
                s_in.wait_event(ev_c[k])
            st["x"][k][:n].copy_(pages_host[b0:b1], non_blocking=True)
            ev_in = torch.cuda.Event()
            ev_in.record(s_in)
        with torch.cuda.stream(s_c):
            s_c.wait_event(ev_in)
            if ev_o[k] is not None:
                s_c.wait_event(ev_o[k])
            xin = engine.normalize_u8(st["x"][k][:n], out=st["xn"][k][:n]) if u8 else st["x"][k][:n]
            engine.forward(xin, out=st["lg"][k][:n])
            front = {name: t[:n] for name, t in st["front"][k].items()}
            engine.text_front(st["lg"][k][:n], size, text_threshold, low_text, out=front)
            if tables is not None:
                engine.text_boxes(front, *tables, out={name: t[:n] for name, t in st["down"][k].items()})
            ev_c[k] = torch.cuda.Event()
            ev_c[k].record(s_c)
        with torch.cuda.stream(s_out):
            s_out.wait_event(ev_c[k])
            for name, t in host.items():
                t[b0:b1].copy_(st["down"][k][name][:n], non_blocking=True)
            ev_o[k] = torch.cuda.Event()
            ev_o[k].record(s_out)
    cur.wait_stream(s_out)
    cur.wait_stream(s_c)
    if sync:
        for ev in ev_o:
            if ev is not None:
                ev.synchronize()
    return host


def detect_text_front_host(engine: DetEngine, pages_host: torch.Tensor, chunk: int = 8, out_size: Tuple[int, int] | None = None,
                           text_threshold: float = 0.6, low_text: float = 0.35, sync: bool = True):
    """Host-to-host detection with the post-processing front half on the device: pinned NCHW pages (or uint8 NHWC pages) in, per
    page the 16-bit text map, the binarised mask and the dynamic thresholds out (3 bytes per pixel over PCIe instead of the 8 of
    two fp32 heat maps; same three-stream pipeline as detect_pages_host).  Returns pinned tensors {"map": [B,H,W],
    "mask": [B,H,W] u8, "thr": [B,4]}; feed them to text_boxes_from_front()."""
    return _front_pipeline(engine, pages_host, chunk, out_size, text_threshold, low_text, sync)


def detect_text_boxes_host(engine: DetEngine, pages_host: torch.Tensor, chunk: int = 8, out_size: Tuple[int, int] | None = None,
                           text_threshold: float = 0.6, low_text: float = 0.35, max_boxes: int = DEFAULT_MAX_BOXES,
                           max_points: int = DEFAULT_MAX_POINTS):
    """Host-to-host detection with the whole text-box post-processing of detect_boxes (surya/detection/heatmap.py:27-107) on the
    device except cv2.minAreaRect: pages in as for detect_text_front_host, per page (list of 4x2 float32 boxes, list of
    confidences) out, equal to text_boxes_from_front on detect_text_front_host's output.  Only the box tables cross PCIe
    (max_boxes * 32 + max_points * 8 + 8 bytes per page).  A page whose components exceed the table capacity is run again through
    the text front and finished on the host by text_boxes_from_front.  The host finish runs in the calling thread: it is mostly
    Python, and a thread pool over the pages was slower."""
    tabs = _front_pipeline(engine, pages_host, chunk, out_size, text_threshold, low_text, True, (max_boxes, max_points))
    count, overflow, box, peak, points = (tabs[k].numpy() for k in ("count", "overflow", "box", "peak", "points"))
    out = [None if overflow[b] else text_boxes_from_tables(box[b], peak[b], points[b], int(count[b])) for b in range(len(count))]
    over = [b for b in range(len(count)) if overflow[b]]
    if over:
        front = detect_text_front_host(engine, pages_host[over].pin_memory(), chunk, out_size, text_threshold, low_text)
        maps = front["map"] if front["map"].dtype != torch.bfloat16 else front["map"].float()
        for j, b in enumerate(over):
            out[b] = text_boxes_from_front(maps[j].numpy(), front["mask"][j].numpy(), float(front["thr"][j, 0]),
                                           float(front["thr"][j, 1]))
    return out


def text_boxes_from_front(line_map, mask, text_threshold: float, low_text: float):
    """Back half of detect_boxes (surya/detection/heatmap.py:33-107) on the host, fed by the device-side front half: connected
    components of the binarised mask, size / peak filtering, dilation, minimum-area rectangle, diamond fix-up, clockwise order,
    confidences normalised by the page maximum.  line_map: [H, W] 16-bit or fp32 map, mask: [H, W] uint8, thresholds as computed
    on the device for this page.  Returns (list of 4x2 float32 boxes, list of confidences) exactly like detect_boxes."""
    import cv2
    import numpy as np

    linemap = np.asarray(line_map)
    if linemap.dtype != np.float32:
        linemap = linemap.astype(np.float32)
    img_h, img_w = linemap.shape
    label_count, labels, stats, _ = cv2.connectedComponentsWithStats(np.ascontiguousarray(mask), connectivity=4)
    det, confidences, max_confidence = [], [], 0
    for k in range(1, label_count):
        if stats[k, cv2.CC_STAT_AREA] < 10:
            continue
        x, y, w, h = stats[k, [cv2.CC_STAT_LEFT, cv2.CC_STAT_TOP, cv2.CC_STAT_WIDTH, cv2.CC_STAT_HEIGHT]]
        niter = int(np.sqrt(min(w, h)))
        buffer = 1
        sx, sy = max(0, x - niter - buffer), max(0, y - niter - buffer)
        ex, ey = min(img_w, x + w + niter + buffer), min(img_h, y + h + niter + buffer)
        comp = labels[sy:ey, sx:ex] == k
        line_max = np.max(linemap[sy:ey, sx:ex][comp])
        if line_max < text_threshold:
            continue
        ksize = buffer + niter
        seg = cv2.dilate(comp.astype(np.uint8), cv2.getStructuringElement(cv2.MORPH_RECT, (ksize, ksize)))
        y_inds, x_inds = np.nonzero(seg)
        contours = np.column_stack((x_inds + sx, y_inds + sy))
        box = cv2.boxPoints(cv2.minAreaRect(contours))
        bw, bh = np.linalg.norm(box[0] - box[1]), np.linalg.norm(box[1] - box[2])
        if abs(1 - max(bw, bh) / (min(bw, bh) + 1e-5)) <= 0.1:
            left, right = contours[:, 0].min(), contours[:, 0].max()
            top, bottom = contours[:, 1].min(), contours[:, 1].max()
            box = np.array([[left, top], [right, top], [right, bottom], [left, bottom]], dtype=np.float32)
        box = np.roll(box, 4 - box.sum(axis=1).argmin(), 0)
        max_confidence = max(max_confidence, line_max)
        confidences.append(line_max)
        det.append(box)
    if max_confidence > 0:
        confidences = [c / max_confidence for c in confidences]
    return det, confidences


def text_boxes_from_tables(box, peak, points, count: int):
    """Host finish of one page's sb_det_text_boxes tables: the part of detect_boxes (surya/detection/heatmap.py:53-107) after
    the dilation, with text_boxes_from_front's types and order.  minAreaRect over two points per dilated row gives the same
    rectangle as over every dilated pixel; the dilated bounding box is the diamond fix-up's left / right / top / bottom."""
    import cv2
    import numpy as np

    det, confidences, max_confidence = [], [], 0
    for k in range(count):
        x0, y0, x1, y1, off, n = (int(v) for v in box[k, :6])
        contours = points[off:off + n].astype(np.int64)       # the dtype np.nonzero gives the host path
        rect = cv2.boxPoints(cv2.minAreaRect(contours))
        bw, bh = np.linalg.norm(rect[0] - rect[1]), np.linalg.norm(rect[1] - rect[2])
        if abs(1 - max(bw, bh) / (min(bw, bh) + 1e-5)) <= 0.1:
            rect = np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], dtype=np.float32)
        rect = np.roll(rect, 4 - rect.sum(axis=1).argmin(), 0)
        line_max = peak[k]
        max_confidence = max(max_confidence, line_max)
        confidences.append(line_max)
        det.append(rect)
    if max_confidence > 0:
        confidences = [c / max_confidence for c in confidences]
    return det, confidences


@dataclass
class PageDetection:
    """Text lines of one page as DetectionPredictor.__call__ reports them (parallel_get_boxes, surya/detection/heatmap.py:156-186):
    polygons and confidences in page coordinates, image_bbox = [0, 0, width, height], and the stitched heatmap's (width, height)."""
    polygons: List[List[List[int]]]
    confidences: List[float]
    image_bbox: List[int]
    heatmap_size: Tuple[int, int]


def _page_groups(sizes, ph: int, chunk: int) -> List[List[int]]:
    """Consecutive pages whose chunks fit one device round of at most `chunk` chunks (a page with more chunks goes alone)."""
    from .page_prep import split_plan

    groups, cur, n = [], [], 0
    for i, (_, h) in enumerate(sizes):
        k = len(split_plan(h, ph))
        if cur and n + k > chunk:
            groups.append(cur)
            cur, n = [], 0
        cur.append(i)
        n += k
    if cur:
        groups.append(cur)
    return groups


def detect_text_pages(engine: DetEngine, pages, processor_size: Tuple[int, int], chunk: int = 16, text_threshold: float = 0.6,
                      low_text: float = 0.35, max_boxes: int = DEFAULT_MAX_BOXES, max_points: int = DEFAULT_MAX_POINTS,
                      max_chunks: int | None = None, max_page_pixels: int | None = None) -> List[PageDetection]:
    """DetectionPredictor.__call__ (surya/detection/__init__.py:27-151 + parallel_get_boxes) for uint8 RGB pages [h, w, 3] of any
    size, everything up to the minimum-area rectangles on the device: the pages go up as they are (3 bytes per pixel, one packed
    pinned upload per round), sb_det_page_resize cuts tall pages into chunks and resizes them exactly like split_image +
    prepare_image, the engine runs on the chunks, sb_det_text_front_stitched stitches each page's chunk heatmaps and thresholds
    the whole page, sb_det_text_boxes extracts its lines at the page's stitched height.  processor_size = (width, height), a
    multiple of 32 within the engine's max_hw.  Raises SuryaB200Error for a page beyond max_page_pixels or max_chunks."""
    import numpy as np

    from . import page_prep as pp
    from .pipeline import page_polygons

    pw, ph = processor_size
    if ph > engine.max_hw[0] or pw > engine.max_hw[1] or ph % 32 or pw % 32:
        raise _lib.SuryaB200Error(f"processor size {pw}x{ph} must be a multiple of 32 within {engine.max_hw[::-1]}")
    pages = [np.ascontiguousarray(p) for p in pages]
    for i, p in enumerate(pages):
        if p.dtype != np.uint8 or p.ndim != 3 or p.shape[2] != 3:
            raise _lib.SuryaB200Error(f"page {i} must be uint8 [h, w, 3], got {p.dtype} {list(p.shape)}")
    sizes = [(p.shape[1], p.shape[0]) for p in pages]
    limits = {"max_chunks": max_chunks or pp.DEFAULT_MAX_CHUNKS, "max_page_pixels": max_page_pixels or pp.DEFAULT_MAX_PAGE_PIXELS}
    pp.plan_pages(sizes, processor_size, **limits)             # every page is checked before any work starts
    dev = engine.device
    out: List[PageDetection] = []
    for group in _page_groups(sizes, ph, chunk):
        plan = pp.plan_pages([sizes[i] for i in group], processor_size, **limits)
        up = torch.empty((int(plan.page_off[-1]),), dtype=torch.uint8).pin_memory()
        upn = up.numpy()
        for j, i in enumerate(group):
            upn[plan.page_off[j]:plan.page_off[j + 1]] = pages[i].reshape(-1)
        chunks = engine.page_resize(up.to(dev, non_blocking=True), plan, processor_size)
        logits = engine.forward(engine.normalize_u8(chunks))
        front = engine.text_front_stitched(logits, plan, (ph, pw), text_threshold, low_text)
        P = len(group)
        tabs = box_tables(P, max_boxes, max_points, device=dev)
        j = 0
        while j < P:                       # pages of equal stitched height share a launch
            r0, rows = (int(v) for v in plan.page_tab[j])
            k = j + 1
            while k < P and int(plan.page_tab[k, 1]) == rows:
                k += 1
            n = k - j
            sub = {"map": front["map"][r0:r0 + n * rows].view(n, rows, pw), "mask": front["mask"][r0:r0 + n * rows].view(n, rows, pw),
                   "thr": front["thr"][j:k]}
            engine.text_boxes(sub, max_boxes, max_points, out={name: t[j:k] for name, t in tabs.items()})
            j = k
        host = {name: t.cpu() for name, t in tabs.items()}
        thr = front["thr"].cpu()
        for j, i in enumerate(group):
            r0, rows = (int(v) for v in plan.page_tab[j])
            if host["overflow"][j]:             # beyond the table capacity: finish the page on the host from its text front
                boxes, conf = text_boxes_from_front(front["map"][r0:r0 + rows].float().cpu().numpy(),
                                                    front["mask"][r0:r0 + rows].cpu().numpy(), float(thr[j, 0]), float(thr[j, 1]))
            else:
                boxes, conf = text_boxes_from_tables(host["box"][j].numpy(), host["peak"][j].numpy(), host["points"][j].numpy(),
                                                     int(host["count"][j]))
            polys, conf = page_polygons(boxes, conf, sizes[i], (pw, rows))
            out.append(PageDetection(polys, conf, [0, 0, sizes[i][0], sizes[i][1]], (pw, rows)))
    return out
