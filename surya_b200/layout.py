"""Layout path: Donut-Swin encoder + ADETR box decoder on the CUDA kernels, behind the call surface LayoutPredictor uses.

  * LayoutEngine        packed weights + forward passes built from libsurya_b200.so ops (wgmma GEMMs for every Linear,
                        swin_window_attn, layernorm, decode_attn / attn_single_query, ...); round 1 drives the layer loops
                        from Python (correctness first), the kernels are the same ones the C++ engines use
  * B200LayoutModel     quacks like the model LayoutPredictor touches (surya/layout/__init__.py:83-123, 222):
                        model.encoder(pixel_values=...)[0], model.decoder(input_boxes=..., encoder_hidden_states=...,
                        cache_position=..., use_cache=True, prefill=...) -> {"bbox_logits", "class_logits"},
                        model.decoder.model._setup_cache / _clear_cache, config fields
  * layout_greedy       the predictor's device-side loop: encoder once, greedy box decoding (surya/layout/__init__.py:106-183)

No PyTorch math on the forward path (torch = memory + streams), no import of oracle/.
"""
from __future__ import annotations

import ctypes
import math
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


class LayoutEngine:
    GRAPH_GROUP = 8      # decode steps per CUDA-graph replay in run_loop

    def __init__(self, cfg: LayoutConfig, sd_enc: Dict[str, torch.Tensor], sd_dec: Dict[str, torch.Tensor],
                 dtype: torch.dtype = torch.float16, device: str | torch.device = "cuda", max_batch: int = 16,
                 impl: str = "native", s_max: Optional[int] = None, max_rows: int = 0, max_prefill_tokens: int = 0):
        """impl = "native": layer loops, workspaces and the decode loop run inside libsurya_b200.so (sb_layout_*);
        impl = "ops": the same CUDA kernels launched one C-ABI call at a time from this module (kept as the readable statement of
        the op sequence and as a cross-check — results are bit-identical).  Both need the library and a GPU; neither does any
        math in PyTorch.

        Capacities: max_batch pages per encoder call and tables whose K/V cross_kv() holds; s_max self-attention positions
        (default max_boxes + 72 for tables, + 8 for layout); max_rows decoder rows of decode_rows() and max_prefill_tokens prompt
        tokens per prefill chunk (0: max_batch, the sizes run_loop uses)."""
        self.lib = _lib.load()
        if impl not in ("native", "ops"):
            raise ValueError(impl)
        self.impl = impl
        self._h = None
        self.cfg, self.dtype, self.device, self.max_batch = cfg, dtype, torch.device(device), max_batch
        e, d = cfg.encoder, cfg.decoder
        dev = self.device

        def T(x):
            return x.to(dtype).contiguous().to(dev)

        def B32(x):
            return x.to(dtype).float().contiguous().to(dev)

        # ---- Swin encoder
        K = e.num_channels * e.patch_size ** 2
        self.pe_kp = (K + 63) // 64 * 64
        pw = torch.zeros((e.embed_dim, self.pe_kp))
        pw[:, :K] = sd_enc["embeddings.patch_embeddings.projection.weight"].reshape(e.embed_dim, K)
        self.pe_w, self.pe_b = T(pw), B32(sd_enc["embeddings.patch_embeddings.projection.bias"])
        self.pe_ln = (T(sd_enc["embeddings.norm.weight"]), T(sd_enc["embeddings.norm.bias"]))
        gh, gw = e.grid
        self.stages = []
        for s, (depth, nh) in enumerate(zip(e.depths, e.num_heads)):
            C = e.embed_dim * 2 ** s
            st = {"C": C, "nh": nh, "pos": T(_sincos_table(gw // 2 ** s, gh // 2 ** s, C)), "layers": []}
            for b in range(depth):
                p = f"encoder.layers.{s}.blocks.{b}."
                a = p + "attention.self."
                st["layers"].append({
                    "ln1": (T(sd_enc[p + "layernorm_before.weight"]), T(sd_enc[p + "layernorm_before.bias"])),
                    "qkv_w": T(torch.cat([sd_enc[a + "query.weight"], sd_enc[a + "key.weight"], sd_enc[a + "value.weight"]], 0)),
                    "qkv_b": B32(torch.cat([sd_enc[a + "query.bias"], sd_enc[a + "key.bias"], sd_enc[a + "value.bias"]], 0)),
                    "rpb": T(sd_enc[a + "relative_position_bias_table"]),
                    "o_w": T(sd_enc[p + "attention.output.dense.weight"]), "o_b": B32(sd_enc[p + "attention.output.dense.bias"]),
                    "ln2": (T(sd_enc[p + "layernorm_after.weight"]), T(sd_enc[p + "layernorm_after.bias"])),
                    "fc1_w": T(sd_enc[p + "intermediate.dense.weight"]), "fc1_b": B32(sd_enc[p + "intermediate.dense.bias"]),
                    "fc2_w": T(sd_enc[p + "output.dense.weight"]), "fc2_b": B32(sd_enc[p + "output.dense.bias"]),
                    "shift": 0 if b % 2 == 0 else e.window_size // 2,
                })
            if s < len(e.depths) - 1:
                p = f"encoder.layers.{s}.downsample."
                st["merge"] = {"ln": (T(sd_enc[p + "norm.weight"]), T(sd_enc[p + "norm.bias"])), "w": T(sd_enc[p + "reduction.weight"])}
            self.stages.append(st)
        self.enc_pos = T(sd_enc["position_embeddings"][0])

        # ---- ADETR decoder
        nh, nkv, hd, H = d.num_attention_heads, d.num_key_value_heads, d.head_dim, d.hidden_size
        self.kind = d.kind
        if d.kind == "table":
            order = ["w", "h", "cx", "cy", "xskew", "yskew", "x1", "y1", "x3", "y3", "category", "merge", "colspan"]
        else:
            order = list(LAYOUT_EMBED_TABLES) + ["label"]
        self.tables = [T(sd_dec[f"model.embed_tokens.{t}_embed.weight"]) for t in order]
        self.layers = []
        for l in range(d.num_hidden_layers):
            p = f"model.layers.{l}."
            gate, up = sd_dec[p + "mlp_block.gate_proj.weight"], sd_dec[p + "mlp_block.up_proj.weight"]
            self.layers.append({
                "cross_norm": T(sd_dec[p + "cross_pre_norm.weight"]), "self_norm": T(sd_dec[p + "temporal_pre_norm.weight"]),
                "mlp_norm": T(sd_dec[p + "channel_pre_norm.weight"]),
                "cq_w": T(sd_dec[p + "cross_attn_block.q_proj.weight"]),
                "ckv_w": T(torch.cat([sd_dec[p + "cross_attn_block.k_proj.weight"], sd_dec[p + "cross_attn_block.v_proj.weight"]], 0)),
                "co_w": T(sd_dec[p + "cross_attn_block.o_proj.weight"]), "co_b": B32(sd_dec[p + "cross_attn_block.o_proj.bias"]),
                "sqkv_w": T(torch.cat([sd_dec[p + "temporal_block.q_proj.weight"], sd_dec[p + "temporal_block.k_proj.weight"],
                                       sd_dec[p + "temporal_block.v_proj.weight"]], 0)),
                "so_w": T(sd_dec[p + "temporal_block.o_proj.weight"]), "so_b": B32(sd_dec[p + "temporal_block.o_proj.bias"]),
                "gu_w": T(torch.stack([gate, up], 1).reshape(2 * gate.shape[0], gate.shape[1])),
                "down_w": T(sd_dec[p + "mlp_block.down_proj.weight"]),
            })
        self.final_norm = T(sd_dec["model.final_norm.weight"])
        self.out_ln = (T(sd_dec["pre_output_norm.weight"]), T(sd_dec["pre_output_norm.bias"]))
        if d.kind == "table":
            self.head_w = {k: T(sd_dec[f"box_property_heads.{k}.weight"]) for k in TABLE_HEADS}
        else:
            self.cls_w = T(sd_dec["lm_head.weight"])
            self.bbox_w, self.bbox_b = T(sd_dec["bbox_head.weight"]), T(sd_dec["bbox_head.bias"])
        self.inv_freq = (1.0 / (d.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))).to(dev)
        # table prompts carry the query + column boxes
        self.s_max = int(s_max) if s_max is not None else d.max_boxes + (72 if d.kind == "table" else 8)
        self.max_rows = max(int(max_rows), max_batch) if max_rows else max_batch
        self.max_prefill_tokens = max(int(max_prefill_tokens), self.max_rows)
        self._row_max_rows, self._row_max_prefill = int(max_rows), int(max_prefill_tokens)
        if impl == "native":
            self._create_native()
        self._cache_batch = 0
        self._ckv: List[Optional[torch.Tensor]] = [None] * d.num_hidden_layers
        self.kcache: List[torch.Tensor] = []
        self.vcache: List[torch.Tensor] = []
        self.n_enc = 0

    # ---------------------------------------------------------------------------------------------- native engine
    def _weight_table(self) -> List[torch.Tensor]:
        """Flat device-tensor list in the SB_LW_* order documented in include/surya_b200.h."""
        d = self.cfg.decoder
        w = [self.pe_w, self.pe_b, self.pe_ln[0], self.pe_ln[1], self.enc_pos]
        for st in self.stages:
            w.append(st["pos"])
            for L in st["layers"]:
                w += [L["ln1"][0], L["ln1"][1], L["qkv_w"], L["qkv_b"], L["rpb"], L["o_w"], L["o_b"], L["ln2"][0], L["ln2"][1],
                      L["fc1_w"], L["fc1_b"], L["fc2_w"], L["fc2_b"]]
            if "merge" in st:
                w += [st["merge"]["ln"][0], st["merge"]["ln"][1], st["merge"]["w"]]
        w += list(self.tables)
        for L in self.layers:
            w += [L["cross_norm"], L["self_norm"], L["mlp_norm"], L["cq_w"], L["ckv_w"], L["co_w"], L["co_b"], L["sqkv_w"],
                  L["so_w"], L["so_b"], L["gu_w"], L["down_w"]]
        w += [self.final_norm, self.out_ln[0], self.out_ln[1], self.inv_freq]
        if self.kind == "table":
            w += [self.head_w[k] for k in TABLE_HEADS]
        else:
            w += [self.bbox_w, self.bbox_b, self.cls_w]
        return w

    def _create_native(self):
        e, d = self.cfg.encoder, self.cfg.decoder
        c = _LayoutCfgC()
        c.dtype = ops.dt_code(self.dtype)
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
        head_n = [d.category_count, d.merge_count, 1, d.header_count] if d.kind == "table" else [d.label_count]
        c.n_out_heads = len(head_n)
        for i, n in enumerate(head_n):
            c.head_n[i] = n
        c.eos, c.pad = d.eos_token_id, d.pad_token_id
        c.max_batch, c.s_max = self.max_batch, self.s_max
        c.max_rows, c.max_prefill_tokens = self._row_max_rows, self._row_max_prefill
        self._wt = self._weight_table()          # keeps the device tensors alive
        arr = (ctypes.c_void_p * len(self._wt))(*[t.data_ptr() for t in self._wt])
        self._h = ctypes.c_void_p()
        self.lib.sb_layout_workspace_bytes.restype = ctypes.c_size_t
        with torch.cuda.device(self.device):
            _lib.check(self.lib.sb_layout_create(ctypes.byref(c), arr, ctypes.c_int(len(self._wt)), ctypes.byref(self._h)),
                       "sb_layout_create")
        self._head_n = head_n

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
        """DonutSwinLayoutModel.forward (surya/layout/model/encoder.py:33-81): NCHW pixels -> [B, L, hidden]."""
        e = self.cfg.encoder
        B, _, Hi, Wi = pixel_values.shape
        if self.impl == "native" and B > 0:
            if (Hi, Wi) != tuple(e.image_size):
                raise _lib.SuryaB200Error(f"layout encoder expects {e.image_size} inputs, got {(Hi, Wi)}")
            if not pixel_values.is_cuda:
                pixel_values = pixel_values.to(self.device, non_blocking=True)
            if pixel_values.dtype not in (torch.float32, self.dtype):
                raise _lib.SuryaB200Error("pixel_values must be float32 or the engine dtype")
            pixel_values = pixel_values.contiguous()
            gh, gw = e.grid
            Lk = (gh >> (len(e.depths) - 1)) * (gw >> (len(e.depths) - 1))
            out = torch.empty((B, Lk, e.hidden_size), dtype=self.dtype, device=self.device)
            for b0 in range(0, B, self.max_batch):
                b1 = min(B, b0 + self.max_batch)
                _lib.check(self.lib.sb_layout_encode(self._h, _lib.ptr(pixel_values[b0:b1]), ctypes.c_int(1 if pixel_values.dtype == torch.float32 else 0),
                                                     ctypes.c_int(b1 - b0), _lib.ptr(out[b0:b1]), _lib.stream_ptr()), "sb_layout_encode")
            return out
        if B == 0:
            raise _lib.SuryaB200Error("empty batch: the predictors return before calling the model (layout/__init__.py:193-195)")
        if (Hi, Wi) != tuple(e.image_size):
            raise _lib.SuryaB200Error(f"layout encoder expects {e.image_size} inputs, got {(Hi, Wi)}")
        if not pixel_values.is_cuda:
            pixel_values = pixel_values.to(self.device, non_blocking=True)
        if pixel_values.dtype not in (torch.float32, self.dtype):
            raise _lib.SuryaB200Error("pixel_values must be float32 or the engine dtype")
        x = ops.patch_gather(pixel_values, e.patch_size, self.pe_kp, self.dtype)
        x = ops.gemm(x, self.pe_w, bias=self.pe_b)
        x = ops.layernorm(x, *self.pe_ln, eps=1e-5)
        H, W = e.grid
        for st in self.stages:
            C, nh = st["C"], st["nh"]
            ops.add_bcast_rows_(x, st["pos"])
            for L in st["layers"]:
                h = ops.layernorm(x, *L["ln1"], eps=e.layer_norm_eps)
                qkv = ops.gemm(h, L["qkv_w"], bias=L["qkv_b"])
                a = ops.swin_window_attn(qkv, L["rpb"], B, H, W, nh, L["shift"] if min(H, W) > e.window_size else 0, qkv_bias=L["qkv_b"])
                x = ops.gemm(a, L["o_w"], bias=L["o_b"], residual=x)
                h = ops.layernorm(x, *L["ln2"], eps=e.layer_norm_eps)
                h = ops.gemm(h, L["fc1_w"], bias=L["fc1_b"], act="gelu")
                x = ops.gemm(h, L["fc2_w"], bias=L["fc2_b"], residual=x)
            if "merge" in st:
                m = ops.patch_merge_gather(x, B, H, W)
                m = ops.layernorm(m, *st["merge"]["ln"], eps=1e-5)
                x = ops.gemm(m, st["merge"]["w"])
                H, W = H // 2, W // 2
        ops.add_bcast_rows_(x, self.enc_pos[: H * W])
        return x.view(B, H * W, -1)

    # ---------------------------------------------------------------------------------------------- decoder
    def setup_cache(self, batch: int):
        """SuryaADETRDecoderModel._setup_cache (surya/common/adetr/decoder.py): fresh self / cross caches."""
        d = self.cfg.decoder
        self._ckv = [None] * d.num_hidden_layers
        if batch != self._cache_batch:
            shape = (batch, d.num_key_value_heads, self.s_max, d.head_dim)
            self.kcache = [torch.zeros(shape, dtype=self.dtype, device=self.device) for _ in range(d.num_hidden_layers)]
            self.vcache = [torch.zeros(shape, dtype=self.dtype, device=self.device) for _ in range(d.num_hidden_layers)]
            self._cache_batch = batch
        self._slot = torch.arange(batch, dtype=torch.int32, device=self.device)

    def clear_cache(self):
        self._ckv = [None] * self.cfg.decoder.num_hidden_layers

    def decode_step(self, boxes: torch.Tensor, enc: torch.Tensor, position, caches=None):
        """One q_len = 1 decoder call (SuryaLayoutDecoder.forward, surya/layout/model/decoder.py:95-126).
        boxes int64 [B, 7|10]; enc [B, L, Henc]; position = cache position of this token (int, or an int32 device tensor [B]
        when the step is replayed from a CUDA graph).  Returns (bbox sigmoid [B,6] fp32, class logits [B, label_count] fp32
        holding the dtype-rounded values) for layout, the dict of five head outputs for table_rec."""
        d = self.cfg.decoder
        nh, nkv, hd, H = d.num_attention_heads, d.num_key_value_heads, d.head_dim, d.hidden_size
        B, Lk = enc.shape[0], enc.shape[1]
        if not torch.is_tensor(position) and position >= self.s_max:
            raise _lib.SuryaB200Error("decoder position exceeds the allocated self-attention cache")
        kcache, vcache, slot = caches if caches is not None else (self.kcache, self.vcache, self._slot)
        scale = hd ** -0.5
        if self.kind == "table":
            x = ops.label_embed(boxes, self.tables, d.box_embed_size, d.property_embed_size, d.bbox_size, d.vocab_size, self.dtype)
        else:
            x = ops.bbox_embed_sum(boxes, self.tables, H, d.bbox_size, self.dtype)
        pos = position if torch.is_tensor(position) else torch.full((B,), position, dtype=torch.int32, device=self.device)
        enc2d = enc.reshape(B * Lk, -1)
        for l, L in enumerate(self.layers):
            raw = x
            n = ops.rmsnorm_adetr(x, L["cross_norm"], d.rms_norm_eps)
            q = ops.gemm(n, L["cq_w"])
            if self._ckv[l] is None:      # K/V of the encoder states, computed at the first call and cached
                self._ckv[l] = ops.gemm(enc2d, L["ckv_w"])
            a = ops.attn_single_query(q, self._ckv[l], Lk, nh, nkv, hd, scale)
            cross = ops.gemm(a, L["co_w"], bias=L["co_b"], residual=raw)
            n = ops.rmsnorm_adetr(cross, L["self_norm"], d.rms_norm_eps)
            qkv = ops.gemm(n, L["sqkv_w"])
            a = ops.decode_attn(qkv, kcache[l], vcache[l], slot, pos, self.inv_freq, nh, nkv, hd, scale)
            res = ops.gemm(a, L["so_w"], bias=L["so_b"], residual=raw if d.double_residual_flow else cross)
            n = ops.rmsnorm_adetr(res, L["mlp_norm"], d.rms_norm_eps)
            m = ops.gemm(n, L["gu_w"], act="gelu_tanh", swiglu=True)
            x = ops.gemm(m, L["down_w"], residual=res, splitk=True)
        x = ops.rmsnorm_adetr(x, self.final_norm, d.rms_norm_eps)
        h = ops.layernorm(x, *self.out_ln, eps=d.layer_norm_eps)
        if self.kind == "table":     # SuryaTableRecDecoder.forward (surya/table_rec/model/decoder.py:121-155): 5 bias-free heads
            return {k: ops.small_head(h, self.head_w[k], None, sigmoid=(k == "bbox"))[0] for k in TABLE_HEADS}
        bbox, _ = ops.small_head(h, self.bbox_w, self.bbox_b, sigmoid=True)
        cls, _ = ops.small_head(h, self.cls_w, None, sigmoid=False)
        return bbox, cls


    def decode_prompt(self, ids: torch.Tensor, enc: torch.Tensor, start: int = 0):
        """q_len > 1 call (the table query prompt, surya/table_rec/processor.py:68-82): causal self-attention makes the
        batched prefill identical to feeding the tokens one position at a time; only the last position's outputs are used
        by the predictors (table_rec/__init__.py:78)."""
        out = None
        for j in range(ids.shape[1]):
            out = self.decode_step(ids[:, j].contiguous(), enc, start + j)
        return out

    def next_tokens(self, head_out, **loop):
        """Per-step token formation on the device (layout/__init__.py:125-137; table_rec/__init__.py:76-121)."""
        d = self.cfg.decoder
        if self.kind == "table":
            o = head_out
            return ops.box_next_token(o["bbox"], [o["category"], o["merges"], o["colspan"], o["is_header"]], [0, 0, 1, 0],
                                      d.bbox_size, done_head=0, eos=d.eos_token_id, pad=d.pad_token_id, **loop)
        bbox, cls = head_out
        return ops.box_next_token(bbox, [cls], [0], d.bbox_size, **loop)

    # ---------------------------------------------------------------------------------------------- graph-replayed decode loop
    def _loop_state(self, B: int, Lk: int, T: int):
        d = self.cfg.decoder
        st = self._loops.get(B) if hasattr(self, "_loops") else None
        if not hasattr(self, "_loops"):
            self._loops = {}
        if st is not None and st["Lk"] == Lk and st["T"] >= T:
            return st
        dev, ncol = self.device, d.token_width
        shape = (B, d.num_key_value_heads, self.s_max, d.head_dim)
        head_n = [d.category_count, d.merge_count, 1, d.header_count] if self.kind == "table" else [d.label_count]
        st = {"Lk": Lk, "T": T, "graph": None,
              "tok": torch.zeros((B, ncol), dtype=torch.int64, device=dev), "pos": torch.zeros((B,), dtype=torch.int32, device=dev),
              "base": torch.zeros((1,), dtype=torch.int32, device=dev),
              "enc": torch.empty((B, Lk, d.encoder_hidden_size), dtype=self.dtype, device=dev),
              "ckv": [torch.empty((B * Lk, 2 * d.num_key_value_heads * d.head_dim), dtype=self.dtype, device=dev) for _ in self.layers],
              "caches": ([torch.zeros(shape, dtype=self.dtype, device=dev) for _ in self.layers],
                         [torch.zeros(shape, dtype=self.dtype, device=dev) for _ in self.layers],
                         torch.arange(B, dtype=torch.int32, device=dev)),
              "hist": {"tok": torch.zeros((T, B, ncol), dtype=torch.int64, device=dev),
                       "bbox": torch.zeros((T, B, 6), dtype=torch.float32, device=dev),
                       "heads": [torch.zeros((T, B, n), dtype=torch.float32, device=dev) for n in head_n],
                       "done": torch.zeros((T, B), dtype=torch.uint8, device=dev)}}
        self._loops[B] = st
        return st

    def _loop_body(self, st):
        out = self.decode_step(st["tok"], st["enc"], st["pos"], caches=st["caches"])
        self.next_tokens(out, out=st["tok"], cache_pos=st["pos"], hist_base=st["base"], hist=st["hist"])

    def run_loop(self, enc: torch.Tensor, prompt: torch.Tensor, n_steps: int, use_graph: bool = True):
        """The predictors' whole decode pass on the device: prompt prefill, then n_steps greedy tokens with the per-step
        kernels (embedding -> layers -> heads -> token formation + position advance + history append) replayed as ONE CUDA
        graph per step — no host work between steps.  enc [B, Lk, Henc]; prompt int64 [B, q, ncol].
        Returns history views: tokens [n, B, ncol], bbox [n, B, 6], heads (list of [n, B, n_k]), done [n, B]."""
        d = self.cfg.decoder
        B, Lk = enc.shape[0], enc.shape[1]
        q = prompt.shape[1]
        if q - 1 + n_steps > self.s_max:
            raise _lib.SuryaB200Error("prompt + steps exceed the allocated self-attention cache")
        if self.impl == "native":
            if B > self.max_batch:
                raise _lib.SuryaB200Error(f"batch {B} exceeds the engine's max_batch {self.max_batch}")
            hk = (B, n_steps)
            hist = getattr(self, "_nhist", None)
            if hist is None or hist["key"] != hk:       # persistent: same pointers -> the step graphs are reused
                dev, ncol = self.device, d.token_width
                hist = {"key": hk, "tok": torch.zeros((n_steps, B, ncol), dtype=torch.int64, device=dev),
                        "bbox": torch.zeros((n_steps, B, 6), dtype=torch.float32, device=dev),
                        "heads": [torch.zeros((n_steps, B, n), dtype=torch.float32, device=dev) for n in self._head_n],
                        "done": torch.zeros((n_steps, B), dtype=torch.uint8, device=dev)}
                self._nhist = hist
            prompt_d = prompt.to(self.device, torch.int64).contiguous()
            enc_c = enc.contiguous()
            hp = (ctypes.c_void_p * 4)(*([t.data_ptr() for t in hist["heads"]] + [None] * (4 - len(hist["heads"]))))
            _lib.check(self.lib.sb_layout_decode(self._h, _lib.ptr(enc_c), ctypes.c_int(B), _lib.ptr(prompt_d), ctypes.c_int(q),
                                                 ctypes.c_int(n_steps), _lib.ptr(hist["tok"]), _lib.ptr(hist["bbox"]), hp,
                                                 _lib.ptr(hist["done"]), ctypes.c_int(1 if use_graph else 0), _lib.stream_ptr()),
                       "sb_layout_decode")
            return hist["tok"], hist["bbox"], list(hist["heads"]), hist["done"]
        st = self._loop_state(B, Lk, n_steps)
        st["enc"].copy_(enc)
        enc2d = st["enc"].view(B * Lk, -1)
        self._ckv = [ops.gemm(enc2d, L["ckv_w"], out=st["ckv"][l]) for l, L in enumerate(self.layers)]
        prompt = prompt.to(self.device)
        for j in range(q - 1):
            self.decode_step(prompt[:, j].contiguous(), st["enc"], j, caches=st["caches"])
        st["tok"].copy_(prompt[:, q - 1])
        st["pos"].fill_(q - 1)
        st["base"].fill_(q - 1)
        self._loop_body(st)                       # first step eagerly (also warms every kernel before a capture)
        left = n_steps - 1
        if left > 0:
            if use_graph:
                if st["graph"] is None:
                    # two graphs: GROUP steps per replay (one host launch per GROUP decode steps) and a single step for the tail
                    torch.cuda.synchronize(self.device)
                    graphs = {}
                    for k in (self.GRAPH_GROUP, 1):
                        g = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(g):
                            for _ in range(k):
                                self._loop_body(st)
                        graphs[k] = g
                    st["graph"] = graphs          # captures do not execute: positions / history are untouched
                while left >= self.GRAPH_GROUP:
                    st["graph"][self.GRAPH_GROUP].replay()
                    left -= self.GRAPH_GROUP
                for _ in range(left):
                    st["graph"][1].replay()
            else:
                for _ in range(left):
                    self._loop_body(st)
        h = st["hist"]
        return h["tok"][:n_steps], h["bbox"][:n_steps], [x[:n_steps] for x in h["heads"]], h["done"][:n_steps]


    # ---------------------------------------------------------------------------------------------- table_rec two-pass flow
    def cross_kv(self, enc: torch.Tensor):
        """Project and hold the cross-attention K/V of enc [n_tables, Lk, Henc] (n_tables <= max_batch) for decode_rows().
        run_loop() overwrites them: call cross_kv() again before the next decode_rows()."""
        if self.impl != "native":
            raise _lib.SuryaB200Error("cross_kv / decode_rows need the native engine (impl='native')")
        if self.kind != "table":
            raise _lib.SuryaB200Error("cross_kv / decode_rows need a table_rec engine")
        n = enc.shape[0]
        if n < 1 or n > self.max_batch:
            raise _lib.SuryaB200Error(f"{n} tables need max_batch >= {n} (engine has {self.max_batch})")
        enc_c = enc.to(self.device, self.dtype).contiguous()
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
        if self.impl != "native" or self.kind != "table":
            raise _lib.SuryaB200Error("decode_rows needs a native table_rec engine")
        d = self.cfg.decoder
        hk = (rows, n_steps)
        hist = getattr(self, "_rhist", None)
        if hist is None or hist["key"] != hk:       # persistent: same pointers -> the step graphs are reused
            dev, ncol = self.device, d.token_width
            hist = {"key": hk, "tok": torch.zeros((n_steps, rows, ncol), dtype=torch.int64, device=dev),
                    "bbox": torch.zeros((n_steps, rows, 6), dtype=torch.float32, device=dev),
                    "heads": [torch.zeros((n_steps, rows, n), dtype=torch.float32, device=dev) for n in self._head_n],
                    "done": torch.zeros((n_steps, rows), dtype=torch.uint8, device=dev)}
            self._rhist = hist
        prompt_d = prompt.to(self.device, torch.int64).contiguous()
        tab = (ctypes.c_int * rows)(*table)
        hp = (ctypes.c_void_p * 4)(*([t.data_ptr() for t in hist["heads"]] + [None] * (4 - len(hist["heads"]))))
        n_run = ctypes.c_int(0)
        _lib.check(self.lib.sb_layout_decode_rows(self._h, tab, ctypes.c_int(rows), _lib.ptr(prompt_d), ctypes.c_int(q),
                                                  ctypes.c_int(n_steps), _lib.ptr(hist["tok"]), _lib.ptr(hist["bbox"]), hp,
                                                  _lib.ptr(hist["done"]), ctypes.byref(n_run), _lib.stream_ptr()),
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
