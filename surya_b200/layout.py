"""Layout path: Donut-Swin encoder + ADETR box decoder on the CUDA engine, behind the call surface LayoutPredictor uses.

  * pack_layout_weights the reference-named state dicts -> the flat SB_LW_* weight table of include/surya_b200.h
  * LayoutEngine        binding of the sb_layout_* engine in libsurya_b200.so: encoder, the predictors' whole greedy loop on
                        the device (run_loop), single decoder steps for the model surface (decode_step / decode_prompt) and
                        table_rec's cell pass over held cross K/V (cross_kv / decode_rows)
  * B200LayoutModel     quacks like the model LayoutPredictor touches (surya/layout/__init__.py:83-123, 222):
                        model.encoder(pixel_values=...)[0], model.decoder(input_boxes=..., encoder_hidden_states=...,
                        cache_position=..., use_cache=True, prefill=...) -> {"bbox_logits", "class_logits"},
                        model.decoder.model._setup_cache / _clear_cache, config fields
  * layout_greedy       the predictor's device-side loop: encoder once, greedy box decoding (surya/layout/__init__.py:106-183)

No PyTorch math on the forward path (torch = memory + streams), no import of oracle/.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional

import torch

from . import _lib, ops
from .config import LayoutConfig
from .synth import LAYOUT_EMBED_TABLES, TABLE_HEADS


class _LayoutCfgC(ctypes.Structure):
    _fields_ = [
        ("dtype", ctypes.c_int),
        ("img_h", ctypes.c_int), ("img_w", ctypes.c_int), ("patch", ctypes.c_int), ("in_ch", ctypes.c_int),
        ("embed_dim", ctypes.c_int), ("n_stages", ctypes.c_int), ("depths", ctypes.c_int * 4), ("heads", ctypes.c_int * 4),
        ("window", ctypes.c_int), ("enc_ln_eps", ctypes.c_float),
        ("kind", ctypes.c_int),
        ("dec_layers", ctypes.c_int), ("hidden", ctypes.c_int), ("inter", ctypes.c_int), ("enc_hidden", ctypes.c_int),
        ("n_heads", ctypes.c_int), ("n_kv", ctypes.c_int), ("head_dim", ctypes.c_int),
        ("rms_eps", ctypes.c_float), ("dec_ln_eps", ctypes.c_float),
        ("double_residual", ctypes.c_int), ("bbox_size", ctypes.c_int), ("vocab", ctypes.c_int), ("box_w", ctypes.c_int),
        ("prop_w", ctypes.c_int),
        ("n_out_heads", ctypes.c_int), ("head_n", ctypes.c_int * 4),
        ("eos", ctypes.c_int), ("pad", ctypes.c_int),
        ("max_batch", ctypes.c_int), ("s_max", ctypes.c_int),
        ("max_rows", ctypes.c_int), ("max_prefill_tokens", ctypes.c_int),
        ("special_tokens", ctypes.c_int), ("skew_scaler", ctypes.c_int),
    ]


def _sincos_table(width: int, height: int, dim: int) -> torch.Tensor:
    """DonutSwinStage.build_2d_sincos_position_embedding (surya/common/donut/encoder.py:736-761), fp32 on the host."""
    gw = torch.arange(int(width), dtype=torch.float32)
    gh = torch.arange(int(height), dtype=torch.float32)
    gw, gh = torch.meshgrid(gw, gh, indexing="ij")
    pos_dim = dim // 4
    omega = 1.0 / (10000.0 ** (torch.arange(pos_dim, dtype=torch.float32) / pos_dim))
    ow = gw.flatten()[..., None] @ omega[None]
    oh = gh.flatten()[..., None] @ omega[None]
    return torch.concat([ow.sin(), ow.cos(), oh.sin(), oh.cos()], dim=1)


def pack_layout_weights(cfg: LayoutConfig, sd_enc: Dict[str, torch.Tensor], sd_dec: Dict[str, torch.Tensor], dtype: torch.dtype,
                        device) -> List[torch.Tensor]:
    """Pack reference-named encoder / decoder state dicts into the SB_LW_* table (see include/surya_b200.h).

    16-bit tensors are rounded once from fp32 (= model.to(dtype)); Linear biases are kept as the fp32 image of the rounded
    16-bit bias so the GEMM epilogue adds exactly the value the reference adds."""
    e, d = cfg.encoder, cfg.decoder

    def T(x):
        return x.to(dtype).contiguous().to(device)

    def B32(x):
        return x.to(dtype).float().contiguous().to(device)

    # ---- Swin encoder
    K = e.num_channels * e.patch_size ** 2
    pw = torch.zeros((e.embed_dim, (K + 63) // 64 * 64))
    pw[:, :K] = sd_enc["embeddings.patch_embeddings.projection.weight"].reshape(e.embed_dim, K)
    w = [T(pw), B32(sd_enc["embeddings.patch_embeddings.projection.bias"]),
         T(sd_enc["embeddings.norm.weight"]), T(sd_enc["embeddings.norm.bias"]), T(sd_enc["position_embeddings"][0])]
    gh, gw = e.grid
    for s, depth in enumerate(e.depths):
        w.append(T(_sincos_table(gw // 2 ** s, gh // 2 ** s, e.embed_dim * 2 ** s)))
        for b in range(depth):
            p = f"encoder.layers.{s}.blocks.{b}."
            a = p + "attention.self."
            w += [T(sd_enc[p + "layernorm_before.weight"]), T(sd_enc[p + "layernorm_before.bias"]),
                  T(torch.cat([sd_enc[a + "query.weight"], sd_enc[a + "key.weight"], sd_enc[a + "value.weight"]], 0)),
                  B32(torch.cat([sd_enc[a + "query.bias"], sd_enc[a + "key.bias"], sd_enc[a + "value.bias"]], 0)),
                  T(sd_enc[a + "relative_position_bias_table"]),
                  T(sd_enc[p + "attention.output.dense.weight"]), B32(sd_enc[p + "attention.output.dense.bias"]),
                  T(sd_enc[p + "layernorm_after.weight"]), T(sd_enc[p + "layernorm_after.bias"]),
                  T(sd_enc[p + "intermediate.dense.weight"]), B32(sd_enc[p + "intermediate.dense.bias"]),
                  T(sd_enc[p + "output.dense.weight"]), B32(sd_enc[p + "output.dense.bias"])]
        if s < len(e.depths) - 1:
            p = f"encoder.layers.{s}.downsample."
            w += [T(sd_enc[p + "norm.weight"]), T(sd_enc[p + "norm.bias"]), T(sd_enc[p + "reduction.weight"])]

    # ---- ADETR decoder
    if d.kind == "table":
        order = ["w", "h", "cx", "cy", "xskew", "yskew", "x1", "y1", "x3", "y3", "category", "merge", "colspan"]
    else:
        order = list(LAYOUT_EMBED_TABLES) + ["label"]
    w += [T(sd_dec[f"model.embed_tokens.{t}_embed.weight"]) for t in order]
    for l in range(d.num_hidden_layers):
        p = f"model.layers.{l}."
        gate, up = sd_dec[p + "mlp_block.gate_proj.weight"], sd_dec[p + "mlp_block.up_proj.weight"]
        w += [T(sd_dec[p + "cross_pre_norm.weight"]), T(sd_dec[p + "temporal_pre_norm.weight"]), T(sd_dec[p + "channel_pre_norm.weight"]),
              T(sd_dec[p + "cross_attn_block.q_proj.weight"]),
              T(torch.cat([sd_dec[p + "cross_attn_block.k_proj.weight"], sd_dec[p + "cross_attn_block.v_proj.weight"]], 0)),
              T(sd_dec[p + "cross_attn_block.o_proj.weight"]), B32(sd_dec[p + "cross_attn_block.o_proj.bias"]),
              T(torch.cat([sd_dec[p + "temporal_block.q_proj.weight"], sd_dec[p + "temporal_block.k_proj.weight"],
                           sd_dec[p + "temporal_block.v_proj.weight"]], 0)),
              T(sd_dec[p + "temporal_block.o_proj.weight"]), B32(sd_dec[p + "temporal_block.o_proj.bias"]),
              T(torch.stack([gate, up], 1).reshape(2 * gate.shape[0], gate.shape[1])),
              T(sd_dec[p + "mlp_block.down_proj.weight"])]
    hd = d.head_dim
    w += [T(sd_dec["model.final_norm.weight"]), T(sd_dec["pre_output_norm.weight"]), T(sd_dec["pre_output_norm.bias"]),
          (1.0 / (d.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))).to(device)]
    if d.kind == "table":
        w += [T(sd_dec[f"box_property_heads.{k}.weight"]) for k in TABLE_HEADS]
    else:
        w += [T(sd_dec["bbox_head.weight"]), T(sd_dec["bbox_head.bias"]), T(sd_dec["lm_head.weight"])]
    return w


def _head_ptrs(heads: List[torch.Tensor]):
    return (ctypes.c_void_p * 4)(*([t.data_ptr() for t in heads] + [None] * (4 - len(heads))))


class LayoutEngine:
    def __init__(self, cfg: LayoutConfig, sd_enc: Dict[str, torch.Tensor], sd_dec: Dict[str, torch.Tensor],
                 dtype: torch.dtype = torch.float16, device: str | torch.device = "cuda", max_batch: int = 16,
                 s_max: Optional[int] = None, max_rows: int = 0, max_prefill_tokens: int = 0):
        """Layer loops, workspaces and the decode loop run inside libsurya_b200.so (sb_layout_*); this class packs the weights
        and binds the entries.

        Capacities: max_batch pages per encoder call, and tables whose K/V cross_kv() holds (so also the batch of the model
        surface's decode_step); s_max self-attention positions (default max_boxes + 72 for tables, + 8 for layout); max_rows
        decoder rows of decode_rows() and max_prefill_tokens prompt tokens per prefill chunk (0: max_batch, the sizes run_loop
        uses)."""
        self.lib = _lib.load()
        self._h = None
        self.cfg, self.dtype, self.device, self.max_batch = cfg, dtype, torch.device(device), max_batch
        e, d = cfg.encoder, cfg.decoder
        self.kind = d.kind
        gh, gw = e.grid
        self.Lk = (gh >> (len(e.depths) - 1)) * (gw >> (len(e.depths) - 1))
        # table prompts carry the query + column boxes
        self.s_max = int(s_max) if s_max is not None else d.max_boxes + (72 if d.kind == "table" else 8)
        self.max_rows = max(int(max_rows), max_batch) if max_rows else max_batch
        self.max_prefill_tokens = max(int(max_prefill_tokens), self.max_rows)
        self._head_n = [d.category_count, d.merge_count, 1, d.header_count] if d.kind == "table" else [d.label_count]
        self._step_kv = False     # the held cross K/V are the ones decode_step projected since setup_cache / clear_cache

        c = _LayoutCfgC()
        c.dtype = ops.dt_code(dtype)
        c.img_h, c.img_w, c.patch, c.in_ch = e.image_size[0], e.image_size[1], e.patch_size, e.num_channels
        c.embed_dim, c.n_stages, c.window, c.enc_ln_eps = e.embed_dim, len(e.depths), e.window_size, e.layer_norm_eps
        for i, (dep, nh) in enumerate(zip(e.depths, e.num_heads)):
            c.depths[i], c.heads[i] = dep, nh
        c.kind = 1 if d.kind == "table" else 0
        c.dec_layers, c.hidden, c.inter, c.enc_hidden = d.num_hidden_layers, d.hidden_size, d.intermediate_size, d.encoder_hidden_size
        c.n_heads, c.n_kv, c.head_dim = d.num_attention_heads, d.num_key_value_heads, d.head_dim
        c.rms_eps, c.dec_ln_eps = d.rms_norm_eps, d.layer_norm_eps
        c.double_residual, c.bbox_size, c.vocab = int(d.double_residual_flow), d.bbox_size, d.vocab_size
        c.box_w, c.prop_w = d.box_embed_size, d.property_embed_size
        c.n_out_heads = len(self._head_n)
        for i, n in enumerate(self._head_n):
            c.head_n[i] = n
        c.eos, c.pad = d.eos_token_id, d.pad_token_id
        c.max_batch, c.s_max = max_batch, self.s_max
        c.max_rows, c.max_prefill_tokens = int(max_rows), int(max_prefill_tokens)
        c.special_tokens, c.skew_scaler = d.special_token_count, d.skew_scaler
        self._wt = pack_layout_weights(cfg, sd_enc, sd_dec, dtype, self.device)     # keeps the device tensors alive
        arr = (ctypes.c_void_p * len(self._wt))(*[t.data_ptr() for t in self._wt])
        self._h = ctypes.c_void_p()
        self.lib.sb_layout_workspace_bytes.restype = ctypes.c_size_t
        with torch.cuda.device(self.device):
            _lib.check(self.lib.sb_layout_create(ctypes.byref(c), arr, ctypes.c_int(len(self._wt)), ctypes.byref(self._h)),
                       "sb_layout_create")

    def close(self):
        if self._h:
            self.lib.sb_layout_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:       # noqa: BLE001 - interpreter shutdown
            pass

    @property
    def workspace_bytes(self) -> int:
        return int(self.lib.sb_layout_workspace_bytes(self._h)) if self._h else 0

    # ---------------------------------------------------------------------------------------------- encoder
    def encode(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """DonutSwinLayoutModel.forward (surya/layout/model/encoder.py:33-81): NCHW pixels -> [B, L, hidden], in chunks of
        max_batch pages."""
        e = self.cfg.encoder
        B, _, Hi, Wi = pixel_values.shape
        if B == 0:
            raise _lib.SuryaB200Error("empty batch: the predictors return before calling the model (layout/__init__.py:193-195)")
        if (Hi, Wi) != tuple(e.image_size):
            raise _lib.SuryaB200Error(f"layout encoder expects {e.image_size} inputs, got {(Hi, Wi)}")
        if not pixel_values.is_cuda:
            pixel_values = pixel_values.to(self.device, non_blocking=True)
        if pixel_values.dtype not in (torch.float32, self.dtype):
            raise _lib.SuryaB200Error("pixel_values must be float32 or the engine dtype")
        pixel_values = pixel_values.contiguous()
        out = torch.empty((B, self.Lk, e.hidden_size), dtype=self.dtype, device=self.device)
        for b0 in range(0, B, self.max_batch):
            b1 = min(B, b0 + self.max_batch)
            _lib.check(self.lib.sb_layout_encode(self._h, _lib.ptr(pixel_values[b0:b1]), ctypes.c_int(1 if pixel_values.dtype == torch.float32 else 0),
                                                 ctypes.c_int(b1 - b0), _lib.ptr(out[b0:b1]), _lib.stream_ptr()), "sb_layout_encode")
        return out

    def _enc(self, enc: torch.Tensor) -> torch.Tensor:
        """Encoder states as the engine reads them: [n, Lk, enc_hidden] in the engine dtype, contiguous on the device."""
        want = (self.Lk, self.cfg.decoder.encoder_hidden_size)
        if enc.dim() != 3 or tuple(enc.shape[1:]) != want:
            raise _lib.SuryaB200Error(f"encoder states must be [n, {want[0]}, {want[1]}], got {tuple(enc.shape)}")
        return enc.to(self.device, self.dtype).contiguous()

    def _history(self, attr: str, rows: int, n_steps: int) -> dict:
        """History buffers [n_steps, rows, ...] kept on the engine: the same pointers let the engine replay its step graphs."""
        hist = getattr(self, attr, None)
        if hist is None or hist["key"] != (rows, n_steps):
            dev, ncol = self.device, self.cfg.decoder.token_width
            hist = {"key": (rows, n_steps), "tok": torch.zeros((n_steps, rows, ncol), dtype=torch.int64, device=dev),
                    "bbox": torch.zeros((n_steps, rows, 6), dtype=torch.float32, device=dev),
                    "heads": [torch.zeros((n_steps, rows, n), dtype=torch.float32, device=dev) for n in self._head_n],
                    "done": torch.zeros((n_steps, rows), dtype=torch.uint8, device=dev)}
            setattr(self, attr, hist)
        return hist

    # ---------------------------------------------------------------------------------------------- model-surface decoder
    def setup_cache(self, batch: int):
        """SuryaADETRDecoderModel._setup_cache (surya/common/adetr/decoder.py): the next decode_step projects the cross K/V
        of its encoder states; self-attention cache rows 0..batch-1 are written from position 0 on."""
        if batch > self.max_batch:
            raise _lib.SuryaB200Error(f"batch {batch} exceeds the engine's max_batch {self.max_batch}: build the LayoutEngine "
                                      f"with max_batch >= the predictor's batch size")
        self._step_kv = False

    def clear_cache(self):
        self._step_kv = False

    def decode_step(self, boxes: torch.Tensor, enc: torch.Tensor, position: int):
        """One q_len = 1 decoder call (SuryaLayoutDecoder.forward, surya/layout/model/decoder.py:95-126) through sb_layout_step.
        boxes int64 [B, 7|10]; enc [B, L, Henc]; position = cache position of this token.  Returns (bbox sigmoid [B,6] fp32,
        class logits [B, label_count] fp32 holding the dtype-rounded values) for layout, the dict of five head outputs for
        table_rec."""
        if position >= self.s_max:
            raise _lib.SuryaB200Error("decoder position exceeds the allocated self-attention cache")
        if not self._step_kv:      # the encoder K/V, projected at the first call (adetr/decoder.py:150-194) or after run_loop
            self.cross_kv(enc)
            self._step_kv = True
        B = boxes.shape[0]
        tok = boxes.to(self.device, torch.int64).contiguous()
        pos = torch.full((B,), position, dtype=torch.int32, device=self.device)
        bbox = torch.empty((B, 6), dtype=torch.float32, device=self.device)
        heads = [torch.empty((B, n), dtype=torch.float32, device=self.device) for n in self._head_n]
        _lib.check(self.lib.sb_layout_step(self._h, _lib.ptr(tok), _lib.ptr(pos), ctypes.c_int(B), _lib.ptr(bbox), _head_ptrs(heads),
                                           _lib.stream_ptr()), "sb_layout_step")
        if self.kind == "table":
            return dict(zip(TABLE_HEADS, [bbox] + heads))
        return bbox, heads[0]

    def decode_prompt(self, ids: torch.Tensor, enc: torch.Tensor, start: int = 0):
        """q_len > 1 call (the table query prompt, surya/table_rec/processor.py:68-82): causal self-attention makes the
        batched prefill identical to feeding the tokens one position at a time; only the last position's outputs are used
        by the predictors (table_rec/__init__.py:78)."""
        out = None
        for j in range(ids.shape[1]):
            out = self.decode_step(ids[:, j].contiguous(), enc, start + j)
        return out

    # ---------------------------------------------------------------------------------------------- graph-replayed decode loop
    def run_loop(self, enc: torch.Tensor, prompt: torch.Tensor, n_steps: int, use_graph: bool = True):
        """The predictors' whole decode pass on the device: prompt prefill, then n_steps greedy tokens with the per-step
        kernels (embedding -> layers -> heads -> token formation + position advance + history append) replayed as CUDA
        graphs of 8 steps — no host work between steps.  enc [B, Lk, Henc]; prompt int64 [B, q, ncol].  Overwrites the
        cross K/V that cross_kv() holds.
        Returns history views: tokens [n, B, ncol], bbox [n, B, 6], heads (list of [n, B, n_k]), done [n, B]."""
        B, q = enc.shape[0], prompt.shape[1]
        if q - 1 + n_steps > self.s_max:
            raise _lib.SuryaB200Error("prompt + steps exceed the allocated self-attention cache")
        if B > self.max_batch:
            raise _lib.SuryaB200Error(f"batch {B} exceeds the engine's max_batch {self.max_batch}")
        enc_c = self._enc(enc)
        hist = self._history("_nhist", B, n_steps)
        prompt_d = prompt.to(self.device, torch.int64).contiguous()
        self._step_kv = False
        _lib.check(self.lib.sb_layout_decode(self._h, _lib.ptr(enc_c), ctypes.c_int(B), _lib.ptr(prompt_d), ctypes.c_int(q),
                                             ctypes.c_int(n_steps), _lib.ptr(hist["tok"]), _lib.ptr(hist["bbox"]),
                                             _head_ptrs(hist["heads"]), _lib.ptr(hist["done"]), ctypes.c_int(1 if use_graph else 0),
                                             _lib.stream_ptr()),
                   "sb_layout_decode")
        return hist["tok"], hist["bbox"], list(hist["heads"]), hist["done"]

    def run_pages(self, enc: torch.Tensor, page_wh, n_steps: int):
        """LayoutPredictor's decode loop (surya/layout/__init__.py:106-183) on the device through sb_layout_decode_pages: the
        greedy pass of run_loop from the bos prompt, plus the header/footer relabelling of rows whose PageHeader / PageFooter box
        lies away from the edges of their image (page_wh: (w, h) per row, the size the row was preprocessed from) and the stop
        once every row has produced eos / pad.  Returns (tok [n, B, 7], bbox [n, B, 6], class logits [n, B, label_count] with the
        relabelled logit zeroed, done [n, B] = this step's done flag) for the n <= n_steps steps that ran; views of buffers the
        next call overwrites."""
        if self.kind != "layout":
            raise _lib.SuryaB200Error("run_pages needs a layout engine: page sizes drive LayoutPredictor's header/footer rule")
        B = int(enc.shape[0])
        wh = torch.as_tensor(page_wh, dtype=torch.int32).reshape(-1, 2) if not torch.is_tensor(page_wh) else page_wh
        if tuple(wh.shape) != (B, 2):
            raise _lib.SuryaB200Error(f"page_wh must be [{B}, 2] (w, h per row), got {tuple(wh.shape)}")
        if n_steps < 1 or n_steps > self.s_max:
            raise _lib.SuryaB200Error(f"{n_steps} steps need 1 <= n_steps <= s_max {self.s_max}")
        if B < 1 or B > self.max_batch:
            raise _lib.SuryaB200Error(f"batch {B} outside 1..max_batch {self.max_batch}")
        enc_c = self._enc(enc)
        hist = self._history("_phist", B, n_steps)
        if "wh" not in hist:          # persistent: the step graphs read the page sizes through this pointer
            hist["wh"] = torch.zeros((B, 2), dtype=torch.int32, device=self.device)
            hist["bos"] = torch.full((B, 1, 7), self.cfg.decoder.bos_token_id, dtype=torch.int64, device=self.device)
        hist["wh"].copy_(wh.to(torch.int32), non_blocking=False)
        self._step_kv = False
        n_run = ctypes.c_int(0)
        _lib.check(self.lib.sb_layout_decode_pages(self._h, _lib.ptr(enc_c), ctypes.c_int(B), _lib.ptr(hist["bos"]), ctypes.c_int(1),
                                                   _lib.ptr(hist["wh"]), ctypes.c_int(n_steps), _lib.ptr(hist["tok"]),
                                                   _lib.ptr(hist["bbox"]), _lib.ptr(hist["heads"][0]), _lib.ptr(hist["done"]),
                                                   ctypes.byref(n_run), _lib.stream_ptr()),
                   "sb_layout_decode_pages")
        n = n_run.value
        return hist["tok"][:n], hist["bbox"][:n], hist["heads"][0][:n], hist["done"][:n]

    def preprocess(self, pages_dev: torch.Tensor, jobs: torch.Tensor, tap_idx: torch.Tensor, tap_w: torch.Tensor,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """sb_layout_preprocess: uint8 pages packed in pages_dev (device), one job per output image (see layout_pages.plan_jobs)
        -> NCHW pixel values [n_jobs, 3, H, W] in the engine dtype at the encoder size."""
        H, W = self.cfg.encoder.image_size
        n = int(jobs.shape[0])
        if out is None:
            out = torch.empty((n, 3, H, W), dtype=self.dtype, device=self.device)
        if pages_dev.dtype != torch.uint8 or not pages_dev.is_cuda:
            raise _lib.SuryaB200Error("pages must be a uint8 device buffer")
        _lib.check(self.lib.sb_layout_preprocess(ctypes.c_int(ops.dt_code(self.dtype)), _lib.ptr(pages_dev), _lib.ptr(jobs),
                                                 ctypes.c_int(n), _lib.ptr(tap_idx), _lib.ptr(tap_w), ctypes.c_int(H), ctypes.c_int(W),
                                                 _lib.ptr(out), _lib.stream_ptr()), "sb_layout_preprocess")
        return out

    # ---------------------------------------------------------------------------------------------- held cross K/V
    def cross_kv(self, enc: torch.Tensor):
        """Project and hold the cross-attention K/V of enc [n_tables, Lk, Henc] (n_tables <= max_batch) for decode_rows()
        and decode_step().  run_loop() overwrites them: call cross_kv() again before the next decode_rows()."""
        n = enc.shape[0]
        if n < 1 or n > self.max_batch:
            raise _lib.SuryaB200Error(f"{n} tables need max_batch >= {n} (engine has {self.max_batch})")
        enc_c = self._enc(enc)
        self._step_kv = False
        _lib.check(self.lib.sb_layout_cross_kv(self._h, _lib.ptr(enc_c), ctypes.c_int(n), _lib.stream_ptr()), "sb_layout_cross_kv")
        self._held = enc_c          # the projection is stream-ordered: keep its input alive until the next call
        return self

    def decode_rows(self, row_table, prompt: torch.Tensor, n_steps: int):
        """Greedy decode of rows against the K/V held by cross_kv(): row r attends to table row_table[r].  prompt int64
        [rows, q, 10]: positions 0..q-2 are prefilled in one batched pass, then q's last token and n_steps-1 generated tokens
        are decoded, stopping early once every row has produced eos / pad.  Returns (tok [n, rows, 10], bbox [n, rows, 6],
        heads [list of [n, rows, n_k]], done [n, rows]) for the n <= n_steps steps that ran (n >= the step at which the last
        row became done; n_steps when some row never does)."""
        rows, q = int(prompt.shape[0]), int(prompt.shape[1])
        table = [int(t) for t in (row_table.tolist() if torch.is_tensor(row_table) else row_table)]
        if len(table) != rows:
            raise _lib.SuryaB200Error(f"row_table has {len(table)} entries for {rows} prompt rows")
        if rows < 1 or rows > self.max_rows:
            raise _lib.SuryaB200Error(f"{rows} rows need max_rows >= {rows} (engine has {self.max_rows})")
        if q < 1 or n_steps < 1 or q - 1 + n_steps > self.s_max:
            raise _lib.SuryaB200Error(f"a {q}-token prompt and {n_steps} steps need s_max >= {q - 1 + n_steps} (engine has {self.s_max})")
        if q - 1 > self.max_prefill_tokens:
            raise _lib.SuryaB200Error(f"a {q}-token prompt needs max_prefill_tokens >= {q - 1} (engine has {self.max_prefill_tokens})")
        if self.kind != "table":
            raise _lib.SuryaB200Error("decode_rows needs a table_rec engine")
        hist = self._history("_rhist", rows, n_steps)
        prompt_d = prompt.to(self.device, torch.int64).contiguous()
        tab = (ctypes.c_int * rows)(*table)
        n_run = ctypes.c_int(0)
        _lib.check(self.lib.sb_layout_decode_rows(self._h, tab, ctypes.c_int(rows), _lib.ptr(prompt_d), ctypes.c_int(q),
                                                  ctypes.c_int(n_steps), _lib.ptr(hist["tok"]), _lib.ptr(hist["bbox"]),
                                                  _head_ptrs(hist["heads"]), _lib.ptr(hist["done"]), ctypes.byref(n_run),
                                                  _lib.stream_ptr()),
                   "sb_layout_decode_rows")
        n = n_run.value
        return hist["tok"][:n], hist["bbox"][:n], [h[:n] for h in hist["heads"]], hist["done"][:n]


class _Ns:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class B200LayoutModel:
    """Attribute-compatible with what LayoutPredictor uses on `self.model` (surya/layout/__init__.py:83-123, 154-157, 222)."""

    def __init__(self, engine: LayoutEngine):
        self.engine = engine
        self.device, self.dtype = engine.device, engine.dtype
        d = engine.cfg.decoder
        dec_cfg = _Ns(**engine.cfg.decoder.__dict__)
        self.config = _Ns(decoder=dec_cfg, encoder=_Ns(**engine.cfg.encoder.__dict__))
        outer = self

        class _Inner:
            def _setup_cache(self, config, batch, device, dtype):
                outer.engine.setup_cache(batch)

            def _clear_cache(self):
                outer.engine.clear_cache()

        class _Decoder:
            config = dec_cfg
            model = _Inner()

            def __call__(self, input_boxes=None, encoder_hidden_states=None, cache_position=None, use_cache=True, prefill=False, **kw):
                if input_boxes.shape[1] != 1:
                    raise NotImplementedError("pause tokens (q_len > 1) are not used by the shipped config (pause_token_count = 0)")
                if prefill:
                    outer.engine.setup_cache(input_boxes.shape[0])
                bbox, cls = outer.engine.decode_step(input_boxes[:, 0].to(torch.int64), encoder_hidden_states,
                                                     int(cache_position[-1]))
                return {"bbox_logits": bbox.to(outer.dtype).unsqueeze(1), "class_logits": cls.to(outer.dtype).unsqueeze(1)}

        self.decoder = _Decoder()

    def encoder(self, pixel_values=None, **kw):
        return (self.engine.encode(pixel_values),)

    def to(self, *a, **k):
        return self

    def eval(self):
        return self


def layout_greedy(engine: LayoutEngine, pixel_values: torch.Tensor, steps: int, use_graph: bool = True):
    """Device part of LayoutPredictor.batch_layout_detection (surya/layout/__init__.py:106-137, 183): encoder once, then
    `steps` greedy decoder calls; next input = [trunc(bbox * bbox_size) x 6, argmax class].  Returns tokens [B, steps, 7],
    bbox [B, steps, 6] and class logits [B, steps, label_count] (fp32 tensors on the device) and the encoder states."""
    d = engine.cfg.decoder
    enc = engine.encode(pixel_values)
    B = enc.shape[0]
    bos = torch.full((B, 1, 7), d.bos_token_id, dtype=torch.int64, device=engine.device)
    tok, bbox, heads, _ = engine.run_loop(enc, bos, steps, use_graph=use_graph)
    return tok.transpose(0, 1).contiguous(), bbox.transpose(0, 1).contiguous(), heads[0].transpose(0, 1).contiguous(), enc


class B200TableRecModel:
    """Attribute-compatible with what TableRecPredictor uses on `self.model` (surya/table_rec/__init__.py:56-87, 182):
    model.encoder(pixel_values=).last_hidden_state; model.decoder(input_ids=i64[B,q,10], encoder_hidden_states=,
    cache_position=, use_cache=True, prefill=) -> {"box_property_logits": {k: [B,1,n_k]}}; _setup_cache; config ids."""

    def __init__(self, engine: LayoutEngine):
        if engine.kind != "table":
            raise _lib.SuryaB200Error("B200TableRecModel needs an engine built from a table_rec config")
        self.engine = engine
        self.device, self.dtype = engine.device, engine.dtype
        dec_cfg = _Ns(**engine.cfg.decoder.__dict__)
        self.config = _Ns(decoder=dec_cfg, encoder=_Ns(**engine.cfg.encoder.__dict__))
        outer = self

        class _Inner:
            def _setup_cache(self, config, batch, device, dtype):
                outer.engine.setup_cache(batch)

            def _clear_cache(self):
                outer.engine.clear_cache()

        class _Decoder:
            config = dec_cfg
            model = _Inner()

            def __call__(self, input_ids=None, encoder_hidden_states=None, cache_position=None, use_cache=True, prefill=False, **kw):
                if prefill:
                    outer.engine.setup_cache(input_ids.shape[0])
                out = outer.engine.decode_prompt(input_ids.to(torch.int64), encoder_hidden_states, int(cache_position[0]))
                return {"box_property_logits": {k: v.to(outer.dtype).unsqueeze(1) for k, v in out.items()}}

        self.decoder = _Decoder()

    def encoder(self, pixel_values=None, **kw):
        return _Ns(last_hidden_state=self.engine.encode(pixel_values))

    def to(self, *a, **k):
        return self

    def eval(self):
        return self


def table_greedy(engine: LayoutEngine, pixel_values: torch.Tensor, prompt: torch.Tensor, steps: int, use_graph: bool = True):
    """Device part of TableRecPredictor's row/column pass (surya/table_rec/__init__.py:33-131, 180-190): encoder once, prompt
    prefill, `steps` greedy tokens.  Returns tokens [B, steps, 10], done [B, steps] (uint8), per-step head outputs, enc."""
    enc = engine.encode(pixel_values)
    tok, bbox, heads, done = engine.run_loop(enc, prompt, steps, use_graph=use_graph)
    hs = {"bbox": bbox.transpose(0, 1).contiguous()}
    for k, h in zip(("category", "merges", "colspan", "is_header"), heads):
        hs[k] = h.transpose(0, 1).contiguous()
    return tok.transpose(0, 1).contiguous(), done.transpose(0, 1).contiguous(), hs, enc
