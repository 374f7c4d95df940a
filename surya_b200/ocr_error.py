"""ocr_error path on the GPU (SURVEY §8 f4): DistilBertForSequenceClassification forward + the predictor's label loop.

Reference: surya/ocr_error/model/encoder.py:48-91 (Embeddings), :133-195 (MultiHeadSelfAttention), :381-399 (FFN), :408-463
(TransformerBlock), :731-763 (classification head), surya/ocr_error/__init__.py:19-62 (OCRErrorPredictor).  The tokenizer
(surya/ocr_error/tokenizer.py) is host string processing and stays the reference's own.

GPU-first layout: the right-padded [B, L] batch the tokenizer produces (padding="longest") is PACKED on the host — only real
tokens become rows, every text is one segment of the block-diagonal attention kernel, so no pad position is ever embedded,
projected or attended (the reference computes them and masks the keys, encoder.py:171-175).  Per layer: one fused q/k/v GEMM
(wgmma), `attn_varlen` (non-causal), out_lin GEMM with the residual in its epilogue, LayerNorm, lin1 GEMM + erf-GELU epilogue,
lin2 GEMM + residual, LayerNorm; then the [CLS] rows are gathered, pre_classifier GEMM + ReLU epilogue and the 2-way classifier.
Everything launches hand-written sm_90a kernels through the C ABI (`ops.py`); there is no PyTorch fallback.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib, ops
from .config import OcrErrorConfig

ID2LABEL = {0: "good", 1: "bad"}     # surya/ocr_error/model/config.py:8-11


def pack_ocr_error_weights(cfg: OcrErrorConfig, sd: Dict[str, torch.Tensor], dtype: torch.dtype, device) -> Dict[str, object]:
    """Reference-named fp32 state dict -> device tensors in the layouts the kernels read: nn.Linear weights [N, K] K-major in the
    model dtype (q/k/v rows concatenated), Linear biases as fp32 images of the rounded 16-bit bias (the epilogue adds them to the
    fp32 accumulator), LayerNorm / embedding / classifier tensors in the model dtype."""
    def t16(name):
        return sd[name].to(dtype).to(device).contiguous()

    def bias(name):
        return sd[name].to(dtype).to(torch.float32).to(device).contiguous()

    e = "distilbert.embeddings."
    w = {"word": t16(e + "word_embeddings.weight"), "pos": t16(e + "position_embeddings.weight"),
         "emb_ln_w": t16(e + "LayerNorm.weight"), "emb_ln_b": t16(e + "LayerNorm.bias"), "layers": []}
    for i in range(cfg.n_layers):
        b = f"distilbert.transformer.layer.{i}."
        a = b + "attention."
        w["layers"].append({
            "qkv_w": torch.cat([sd[a + n + ".weight"] for n in ("q_lin", "k_lin", "v_lin")], 0).to(dtype).to(device).contiguous(),
            "qkv_b": torch.cat([sd[a + n + ".bias"] for n in ("q_lin", "k_lin", "v_lin")], 0).to(dtype).to(torch.float32).to(device).contiguous(),
            "o_w": t16(a + "out_lin.weight"), "o_b": bias(a + "out_lin.bias"),
            "ln1_w": t16(b + "sa_layer_norm.weight"), "ln1_b": t16(b + "sa_layer_norm.bias"),
            "w1": t16(b + "ffn.lin1.weight"), "b1": bias(b + "ffn.lin1.bias"),
            "w2": t16(b + "ffn.lin2.weight"), "b2": bias(b + "ffn.lin2.bias"),
            "ln2_w": t16(b + "output_layer_norm.weight"), "ln2_b": t16(b + "output_layer_norm.bias"),
        })
    w["pre_w"], w["pre_b"] = t16("pre_classifier.weight"), bias("pre_classifier.bias")
    w["cls_w"], w["cls_b"] = t16("classifier.weight"), t16("classifier.bias")
    return w


def build_pack_plan(input_ids: np.ndarray, attention_mask: Optional[np.ndarray], cfg: OcrErrorConfig) -> Dict[str, np.ndarray]:
    """Host index plan for one right-padded batch: packed token ids, their positions (Embeddings uses arange(L), encoder.py:80),
    per-text segment start / length and the [CLS] row of every text.  Raises on inputs the packed layout cannot represent the way
    the reference computes them (mask holes / left padding, texts without any token) and on out-of-range ids / positions (the
    reference's nn.Embedding would fail on those too)."""
    ids = np.asarray(input_ids)
    if ids.ndim != 2:
        raise _lib.SuryaB200Error(f"ocr_error: input_ids must be [batch, seq], got shape {ids.shape}")
    B, L = ids.shape
    mask = np.ones((B, L), dtype=np.int64) if attention_mask is None else np.asarray(attention_mask)
    if mask.shape != ids.shape:
        raise _lib.SuryaB200Error(f"ocr_error: attention_mask {mask.shape} does not match input_ids {ids.shape}")
    if L > cfg.max_position_embeddings:
        raise _lib.SuryaB200Error(f"ocr_error: sequence length {L} exceeds max_position_embeddings={cfg.max_position_embeddings}")
    keep = mask != 0
    lens = keep.sum(axis=1).astype(np.int64)
    if B and (lens == 0).any():
        raise _lib.SuryaB200Error("ocr_error: a text with an all-zero attention_mask (static-cache batch padding, "
                                  "surya/ocr_error/__init__.py:48-52) has no row in the packed layout: pass the un-padded batch")
    if B and not (keep == (np.arange(L)[None, :] < lens[:, None])).all():
        raise _lib.SuryaB200Error("ocr_error: attention_mask must be a right-padded prefix of ones per text (the tokenizer's "
                                  "padding='longest' layout); holes / left padding are not supported")
    packed = ids[keep].astype(np.int64)
    if packed.size and (packed.min() < 0 or packed.max() >= cfg.vocab_size):
        raise _lib.SuryaB200Error(f"ocr_error: token id outside [0, {cfg.vocab_size})")
    start = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32) if B else np.zeros(0, np.int32)
    pos = (np.arange(L)[None, :].repeat(B, 0))[keep].astype(np.int32) if B else np.zeros(0, np.int32)
    return {"ids": packed.astype(np.int32), "pos": pos, "seq_start": start, "seq_len": lens.astype(np.int32),
            "n_tok": int(packed.size), "max_len": int(lens.max()) if B else 0, "batch": B}


class B200DistilBert:
    """Mirror of the surface OCRErrorPredictor touches on its model (surya/ocr_error/__init__.py:39-56): `model.device`,
    `model(input_ids, attention_mask=...)` -> object with `.logits` [B, num_labels] in the model dtype; plus `.config` / `.dtype`."""

    def __init__(self, cfg: OcrErrorConfig, state_dict: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float16, device=None):
        _lib.load()                                    # raises without the library / a CUDA device: no fallback
        if cfg.dim % cfg.n_heads or (cfg.dim // cfg.n_heads) not in (32, 64, 80, 96, 128):
            raise _lib.SuryaB200Error(f"ocr_error: head_dim {cfg.dim}/{cfg.n_heads} is not one attn_varlen is built for")
        self.config, self.cfg, self.dtype = cfg, cfg, dtype
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.w = pack_ocr_error_weights(cfg, state_dict, dtype, self.device)

    def eval(self):
        return self

    def _upload(self, arr: np.ndarray) -> torch.Tensor:
        """ONE pinned int32 upload per batch (ids | positions | segment starts | segment lengths) through a grow-only page-locked
        staging buffer; the event keeps the next batch from overwriting it before the asynchronous copy has read it."""
        n = int(arr.size)
        pin = getattr(self, "_pin", None)
        if pin is None or pin.numel() < n:
            pin = torch.empty(max(2 * n, 1 << 16), dtype=torch.int32).pin_memory()
            self._pin, self._pin_ev = pin, torch.cuda.Event()
        else:
            self._pin_ev.synchronize()
        pin.numpy()[:n] = arr
        out = pin[:n].to(self.device, non_blocking=True)
        self._pin_ev.record()
        return out

    def forward_packed(self, plan: Dict[str, np.ndarray], return_hidden: bool = False):
        """Run the network over one packed batch (host plan from build_pack_plan); returns logits [B, num_labels] (model dtype)."""
        cfg, w, dev = self.cfg, self.w, self.device
        B, n_tok = plan["batch"], plan["n_tok"]
        if B == 0:
            return torch.zeros((0, cfg.num_labels), dtype=self.dtype, device=dev)
        D, nh = cfg.dim, cfg.n_heads
        hd = D // nh
        idx = self._upload(np.concatenate([plan["ids"], plan["pos"], plan["seq_start"], plan["seq_len"]]))
        ids, pos = idx[:n_tok], idx[n_tok:2 * n_tok]
        seq_start, seq_len = idx[2 * n_tok:2 * n_tok + B], idx[2 * n_tok + B:]
        x = ops.embed_pos_layernorm(ids, pos, w["word"], w["pos"], w["emb_ln_w"], w["emb_ln_b"], cfg.layer_norm_eps)
        scale = 1.0 / math.sqrt(hd)
        for lw in w["layers"]:
            qkv = ops.gemm(x, lw["qkv_w"], bias=lw["qkv_b"])
            ctx = ops.attn_varlen(qkv[:, 0:D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], seq_start, seq_len, plan["max_len"], nh, nh, hd,
                                  False, scale)
            sa = ops.layernorm(ops.gemm(ctx, lw["o_w"], bias=lw["o_b"], residual=x), lw["ln1_w"], lw["ln1_b"], cfg.layer_norm_eps)
            h = ops.gemm(sa, lw["w1"], bias=lw["b1"], act="gelu")
            x = ops.layernorm(ops.gemm(h, lw["w2"], bias=lw["b2"], residual=sa), lw["ln2_w"], lw["ln2_b"], cfg.layer_norm_eps)
        cls = ops.gather_pad_rows(x, seq_start, D, self.dtype)                       # hidden_state[:, 0] (encoder.py:758)
        pooled = ops.gemm(cls, w["pre_w"], bias=w["pre_b"], act="relu")
        logits, _ = ops.small_head(pooled, w["cls_w"], w["cls_b"], sigmoid=False)     # fp32 image of the 16-bit-rounded logits
        logits = logits.to(self.dtype)
        return (logits, x) if return_hidden else logits

    def __call__(self, input_ids, attention_mask=None, **_):
        ids = input_ids.detach().cpu().numpy() if isinstance(input_ids, torch.Tensor) else np.asarray(input_ids)
        mask = None
        if attention_mask is not None:
            mask = attention_mask.detach().cpu().numpy() if isinstance(attention_mask, torch.Tensor) else np.asarray(attention_mask)
        return SimpleNamespace(logits=self.forward_packed(build_pack_plan(ids, mask, self.cfg)))


def detect_errors(model: B200DistilBert, input_ids, attention_mask, batch_size: int = 64) -> List[str]:
    """Mirror of OCRErrorPredictor.batch_ocr_error_detection after tokenisation (surya/ocr_error/__init__.py:26-62): batches of
    `batch_size` texts (default_batch_sizes["cuda"] = 64), argmax over the two labels, ID2LABEL.  The argmax ids of all batches are
    read back with one D2H copy at the end instead of one `.cpu()` per batch."""
    ids = input_ids.detach().cpu().numpy() if isinstance(input_ids, torch.Tensor) else np.asarray(input_ids)
    mask = attention_mask.detach().cpu().numpy() if isinstance(attention_mask, torch.Tensor) else np.asarray(attention_mask)
    n = ids.shape[0]
    preds = []
    for s in range(0, n, batch_size):
        bi, bm = ids[s:s + batch_size], mask[s:s + batch_size]
        L = int(bm.sum(axis=1).max()) if bi.shape[0] else 0        # the global padding='longest' tail is pure padding for this batch
        preds.append(model.forward_packed(build_pack_plan(bi[:, :max(L, 1)], bm[:, :max(L, 1)], model.cfg)).argmax(dim=1))
    if not preds:
        return []
    return [ID2LABEL[int(p)] for p in torch.cat(preds).cpu().tolist()]


def sharded_error_labels(model, input_ids, attention_mask, batch_size: int = 64, device=None) -> List[str]:
    """Multi-GPU form of detect_errors (SURVEY §8e: texts are independent units): every rank classifies its contiguous share of
    the texts and the argmax ids of ALL texts are all-gathered in text order (one int64 per text on the wire).  Works under any
    torch.distributed backend (NCCL on the GPU box, gloo in tests/test_shard_cpu.py); world size 1 is detect_errors."""
    from . import shard

    ids = input_ids.detach().cpu().numpy() if isinstance(input_ids, torch.Tensor) else np.asarray(input_ids)
    mask = attention_mask.detach().cpu().numpy() if isinstance(attention_mask, torch.Tensor) else np.asarray(attention_mask)
    n = int(ids.shape[0])
    if n == 0:
        return []
    inv = {v: k for k, v in ID2LABEL.items()}

    def run_local(lo, hi):
        labels = detect_errors(model, ids[lo:hi], mask[lo:hi], batch_size)
        return torch.tensor([inv[x] for x in labels], dtype=torch.int64)

    out = shard.sharded_pages(run_local, n, device=device, result_meta=((), torch.int64))
    return [ID2LABEL[int(p)] for p in out.cpu().tolist()]
