"""BERT for pre-training (MLM + NSP heads), base and large.

The reference benchmarks HuggingFace ``BertForPreTraining`` built from ``bert_config.json`` /
``bert_base_config.json`` with the vocabulary padded to a multiple of 8 (30522 -> 30528)
(dear/bert_benchmark.py:72-83).  This is an independent implementation of the same architecture
(same parameter tensors and tying: the MLM decoder shares the word-embedding matrix), written for
Hopper: attention goes through ``scaled_dot_product_attention`` (flash kernels) and the QKV
projections are one fused GEMM.
"""
from __future__ import annotations

from dataclasses import dataclass

import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.bias_gelu import linear_gelu
from ..ops.fused_ln import FusedDropoutAddLayerNorm
from ..ops.tc_gemm import fused_ffn


@dataclass
class BertConfig:
    vocab_size: int = 30522
    hidden_size: int = 1024
    num_hidden_layers: int = 24
    num_attention_heads: int = 16
    intermediate_size: int = 4096
    max_position_embeddings: int = 512
    type_vocab_size: int = 2
    hidden_dropout_prob: float = 0.1
    attention_probs_dropout_prob: float = 0.1
    initializer_range: float = 0.02
    layer_norm_eps: float = 1e-12

    def padded_vocab(self, multiple: int = 8) -> int:
        return (self.vocab_size + multiple - 1) // multiple * multiple


BERT_LARGE = BertConfig()                                   # dear/bert_config.json
BERT_BASE = BertConfig(hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                       intermediate_size=3072)              # dear/bert_base_config.json


class Linear(nn.Linear):
    """``nn.Linear`` (same parameters and state-dict keys) whose call selects what happens to the bias:

    * ``"bias"`` (default): ``x W^T + b``;
    * ``"none"``: ``x W^T`` — the bias is consumed by a downstream fused kernel;
    * ``"gelu"``: ``gelu(x W^T + b)`` with the bias gradient fused into the GELU backward;
    * ``"params"``: returns ``(W, b)`` for an op that takes the raw parameters.

    Every mode goes through ``Module.__call__`` so forward pre-hooks run: the decoupled all-reduce
    engine hangs its "this bucket's all-gather has landed" wait on them
    (parallel/optimizer.py: _make_pre_hook), and a parameter must never be read around them."""

    def forward(self, x, epilogue: str = "bias"):              # type: ignore[override]
        if epilogue == "bias":
            return F.linear(x, self.weight, self.bias)
        if epilogue == "none":
            return F.linear(x, self.weight)
        if epilogue == "gelu":
            return linear_gelu(x, self.weight, self.bias)
        if epilogue == "params":
            return self.weight, self.bias
        raise ValueError("unknown epilogue %r" % (epilogue,))


class BertEmbeddings(nn.Module):
    def __init__(self, c: BertConfig, vocab: int):
        super().__init__()
        self.word_embeddings = nn.Embedding(vocab, c.hidden_size)
        self.position_embeddings = nn.Embedding(c.max_position_embeddings, c.hidden_size)
        self.token_type_embeddings = nn.Embedding(c.type_vocab_size, c.hidden_size)
        self.LayerNorm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.dropout = nn.Dropout(c.hidden_dropout_prob)

    def forward(self, input_ids, token_type_ids=None, position_ids=None):
        B, S = input_ids.shape
        if position_ids is None:
            position_ids = torch.arange(S, device=input_ids.device).unsqueeze(0)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        x = self.word_embeddings(input_ids) + self.position_embeddings(position_ids) + \
            self.token_type_embeddings(token_type_ids)
        return self.dropout(self.LayerNorm(x))


def _sdpa_backend(name):
    if not name:
        return None
    from torch.nn.attention import SDPBackend
    return {"cudnn": SDPBackend.CUDNN_ATTENTION, "efficient": SDPBackend.EFFICIENT_ATTENTION,
            "flash": SDPBackend.FLASH_ATTENTION, "math": SDPBackend.MATH}[name.lower()]


try:
    from torch.nn.attention import SDPBackend as _SDPBackend
    _EFFICIENT = _SDPBackend.EFFICIENT_ATTENTION
except Exception:                      # pragma: no cover - very old torch
    _EFFICIENT = None


class BertSelfAttention(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.nh = c.num_attention_heads
        self.hd = c.hidden_size // c.num_attention_heads
        self.qkv = nn.Linear(c.hidden_size, 3 * c.hidden_size)      # fused Q,K,V projection
        self.p_drop = c.attention_probs_dropout_prob
        # optional pin of the SDPA implementation ("cudnn" | "efficient" | "flash" | "math"); default: PyTorch's choice
        self.backend = _sdpa_backend(os.environ.get("DEAR_SDPA_BACKEND"))

    def forward(self, x, attn_bias):
        B, S, H = x.shape
        # unbind (not indexing): its backward is ONE stack of (dq, dk, dv) instead of three zero-filled
        # [B,S,3,H] buffers, three copies and two adds
        q, k, v = self.qkv(x).view(B, S, 3, self.nh, self.hd).unbind(2)
        p = self.p_drop if self.training else 0.0
        backend = self.backend
        if backend is None and x.is_cuda and S <= 128 and attn_bias is not None and _EFFICIENT is not None:
            # short sequences with a key-padding bias: the memory-efficient kernel instead of cuDNN's 128x128-tile
            # flash backward (tools/bert_ops_bench.py --ops attn compares them)
            backend = _EFFICIENT
        if backend is None:
            o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=attn_bias,
                                               dropout_p=p)
        else:
            with torch.nn.attention.sdpa_kernel(backend):
                o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                   attn_mask=attn_bias, dropout_p=p)
        return o.transpose(1, 2).reshape(B, S, H)


class BertLayer(nn.Module):
    """Post-LN transformer layer.  ``fused_ln``: bias + dropout + add + LayerNorm in one kernel
    (ops/fused_ln.py) and bias + GELU in one kernel (ops/bias_gelu.py), bias gradients fused into their
    backward kernels; ``tc_ffn``: feed-forward block on the wgmma GEMMs with GELU / GELU' in the
    epilogues (ops/tc_gemm.py).  Parameters and state-dict keys are identical in every mode."""

    def __init__(self, c: BertConfig, fused_ln: bool = False, tc_ffn: bool = False):
        super().__init__()
        self.attention = BertSelfAttention(c)
        self.attn_out = Linear(c.hidden_size, c.hidden_size)
        self.intermediate = Linear(c.hidden_size, c.intermediate_size)
        self.output = Linear(c.intermediate_size, c.hidden_size)
        self.fused_ln, self.tc_ffn = fused_ln, tc_ffn
        if fused_ln:
            self.attn_norm = FusedDropoutAddLayerNorm(c.hidden_size, eps=c.layer_norm_eps, p=c.hidden_dropout_prob)
            self.out_norm = FusedDropoutAddLayerNorm(c.hidden_size, eps=c.layer_norm_eps, p=c.hidden_dropout_prob)
        else:
            self.attn_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
            self.out_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
            self.dropout = nn.Dropout(c.hidden_dropout_prob)

    def ffn_tc(self, x):
        w1, b1 = self.intermediate(None, "params")
        w2, b2 = self.output(None, "params")
        return fused_ffn(x, w1, b1, w2, b2)

    def forward(self, x, attn_bias):
        ctx = self.attention(x, attn_bias)
        if self.fused_ln:
            # the two output projections run bias-free; their biases are added inside the fused
            # dropout+add+LayerNorm kernel, whose backward also yields the bias gradients
            x = self.attn_norm(self.attn_out(ctx, "none"), x, self.attn_out.bias)
            if self.tc_ffn:
                return self.out_norm(self.ffn_tc(x), x)
            h = self.intermediate(x, "gelu")
            return self.out_norm(self.output(h, "none"), x, self.output.bias)
        x = self.attn_norm(x + self.dropout(self.attn_out(ctx)))
        f = self.ffn_tc(x) if self.tc_ffn else self.output(F.gelu(self.intermediate(x)))
        return self.out_norm(x + self.dropout(f))


class BertModel(nn.Module):
    def __init__(self, c: BertConfig, vocab: int, fused_ln: bool = False, tc_ffn: bool = False):
        super().__init__()
        self.embeddings = BertEmbeddings(c, vocab)
        self.layers = nn.ModuleList(BertLayer(c, fused_ln, tc_ffn) for _ in range(c.num_hidden_layers))
        self.pooler = nn.Linear(c.hidden_size, c.hidden_size)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, position_ids=None):
        x = self.embeddings(input_ids, token_type_ids, position_ids)
        bias = None
        if attention_mask is not None:
            # additive key-padding bias, broadcast over heads and query positions
            bias = (1.0 - attention_mask[:, None, None, :].to(x.dtype)) * torch.finfo(x.dtype).min
        for layer in self.layers:
            x = layer(x, bias)
        pooled = torch.tanh(self.pooler(x[:, 0]))
        return x, pooled


class BertPreTrainingHeads(nn.Module):
    """MLM head (dense + GELU + LayerNorm, decoder tied to the word embeddings, own bias) and NSP head."""

    def __init__(self, c: BertConfig, vocab: int):
        super().__init__()
        self.transform = nn.Linear(c.hidden_size, c.hidden_size)
        self.transform_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.decoder_bias = nn.Parameter(torch.zeros(vocab))
        self.seq_relationship = nn.Linear(c.hidden_size, 2)

    def forward(self, seq, pooled, word_embedding_weight):
        h = self.transform_norm(F.gelu(self.transform(seq)))
        return F.linear(h, word_embedding_weight, self.decoder_bias), self.seq_relationship(pooled)


class BertForPreTraining(nn.Module):
    def __init__(self, config: BertConfig = BERT_LARGE, pad_vocab_to: int = 8, fused_ln: bool = False,
                 tc_ffn: bool = False):
        super().__init__()
        self.config = config
        self.vocab_size = config.padded_vocab(pad_vocab_to)
        self.bert = BertModel(config, self.vocab_size, fused_ln, tc_ffn)
        self.cls = BertPreTrainingHeads(config, self.vocab_size)
        self.apply(self._init)

    def _init(self, m):
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, 0.0, self.config.initializer_range)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.LayerNorm):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, position_ids=None):
        seq, pooled = self.bert(input_ids, token_type_ids, attention_mask, position_ids)
        return self.cls(seq, pooled, self.bert.embeddings.word_embeddings.weight)


class BertPretrainingCriterion(nn.Module):
    """CE(MLM, ignore_index=-1) + CE(NSP), as dear/bert_benchmark.py:101-112."""

    def __init__(self, vocab_size: int):
        super().__init__()
        self.vocab_size = vocab_size

    def forward(self, prediction_scores, seq_relationship_score, masked_lm_labels, next_sentence_labels):
        mlm = F.cross_entropy(prediction_scores.view(-1, self.vocab_size).float(), masked_lm_labels.view(-1),
                              ignore_index=-1)
        nsp = F.cross_entropy(seq_relationship_score.view(-1, 2).float(), next_sentence_labels.view(-1),
                              ignore_index=-1)
        return mlm + nsp


# ---- checkpoints of the reference's model -----------------------------------------------------------------------------
# The reference trains transformers' ``BertForPreTraining`` (dear/bert_benchmark.py:72-83).  Same architecture, different
# module tree: the three attention projections are one [3H, H] GEMM here, the sub-module names are flatter.

_HF_LAYER = [("attention.output.dense", "attn_out"), ("attention.output.LayerNorm", "attn_norm"),
             ("intermediate.dense", "intermediate"), ("output.dense", "output"), ("output.LayerNorm", "out_norm")]
_HF_TOP = [("bert.pooler.dense", "bert.pooler"), ("cls.predictions.transform.dense", "cls.transform"),
           ("cls.predictions.transform.LayerNorm", "cls.transform_norm"), ("cls.seq_relationship", "cls.seq_relationship")]


def from_hf_state_dict(hf: dict, num_layers: int, vocab_size: int = None) -> dict:
    """State dict of this module tree from one of ``transformers.BertForPreTraining`` (vocabulary rows are zero-padded to
    ``vocab_size`` when the model pads its embedding table to a multiple of 8)."""
    out = {}
    for k in ("word_embeddings.weight", "position_embeddings.weight", "token_type_embeddings.weight", "LayerNorm.weight",
              "LayerNorm.bias"):
        out["bert.embeddings." + k] = hf["bert.embeddings." + k]
    for i in range(num_layers):
        src, dst = "bert.encoder.layer.%d." % i, "bert.layers.%d." % i
        for wb in ("weight", "bias"):
            out[dst + "attention.qkv." + wb] = torch.cat([hf[src + "attention.self.%s.%s" % (n, wb)]
                                                          for n in ("query", "key", "value")], 0)
            for a, b in _HF_LAYER:
                out[dst + b + "." + wb] = hf[src + a + "." + wb]
    for a, b in _HF_TOP:
        for wb in ("weight", "bias"):
            out[b + "." + wb] = hf[a + "." + wb]
    out["cls.decoder_bias"] = hf["cls.predictions.bias"]
    if vocab_size is not None:
        for k in ("bert.embeddings.word_embeddings.weight", "cls.decoder_bias"):
            t = out[k]
            if t.shape[0] < vocab_size:
                out[k] = torch.cat([t, t.new_zeros((vocab_size - t.shape[0],) + tuple(t.shape[1:]))], 0)
    return {k: v.clone() for k, v in out.items()}


def to_hf_state_dict(sd: dict, num_layers: int, vocab_size: int = None) -> dict:
    """The inverse: a state dict ``transformers.BertForPreTraining.load_state_dict`` accepts."""
    out = {}
    for k in ("word_embeddings.weight", "position_embeddings.weight", "token_type_embeddings.weight", "LayerNorm.weight",
              "LayerNorm.bias"):
        out["bert.embeddings." + k] = sd["bert.embeddings." + k]
    for i in range(num_layers):
        src, dst = "bert.layers.%d." % i, "bert.encoder.layer.%d." % i
        for wb in ("weight", "bias"):
            q, k_, v = sd[src + "attention.qkv." + wb].chunk(3, 0)
            for n, t in (("query", q), ("key", k_), ("value", v)):
                out[dst + "attention.self.%s.%s" % (n, wb)] = t
            for a, b in _HF_LAYER:
                out[dst + a + "." + wb] = sd[src + b + "." + wb]
    for a, b in _HF_TOP:
        for wb in ("weight", "bias"):
            out[a + "." + wb] = sd[b + "." + wb]
    emb, bias = sd["bert.embeddings.word_embeddings.weight"], sd["cls.decoder_bias"]
    if vocab_size is not None:
        emb, bias = emb[:vocab_size], bias[:vocab_size]
    out["bert.embeddings.word_embeddings.weight"] = emb
    out["cls.predictions.decoder.weight"] = emb                      # tied
    out["cls.predictions.bias"] = bias
    out["cls.predictions.decoder.bias"] = bias
    return {k: v.clone() for k, v in out.items()}


def bert_large(**kw): return BertForPreTraining(BERT_LARGE, **kw)
def bert_base(**kw): return BertForPreTraining(BERT_BASE, **kw)


def synthetic_batch(batch_size: int, seq_len: int, vocab_size: int, device, seed: int = 0):
    """Random BERT-shaped inputs (token ids, mask, segment ids, NSP label, MLM labels)."""
    g = torch.Generator().manual_seed(seed)
    input_ids = torch.randint(0, min(vocab_size, 30000), (batch_size, seq_len), generator=g)
    attention_mask = torch.ones(batch_size, seq_len, dtype=torch.long)
    token_type_ids = torch.randint(0, 2, (batch_size, seq_len), generator=g)
    nsp = torch.randint(0, 2, (batch_size,), generator=g)
    mlm = torch.full((batch_size, seq_len), -1, dtype=torch.long)
    pick = torch.rand(batch_size, seq_len, generator=g) < 0.15
    mlm[pick] = input_ids[pick]
    return tuple(t.to(device) for t in (input_ids, attention_mask, token_type_ids, nsp, mlm))
