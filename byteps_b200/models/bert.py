"""BERT encoder with the pre-training heads (MLM + NSP): the reference's
bandwidth-bound headline workload (BERT-large, ~335 M parameters,
/root/reference/README.md:36-38)."""
import math
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.attn import _packed_tokens, _stock_varlen, self_attention
from ..ops.fp8 import Fp8Linear, fp8_gelu_mlp
from ..ops.ln import DropoutAddLayerNorm
from ..ops.mlm import gather_labelled
from ..ops.xent import softmax_cross_entropy


@dataclass
class BertConfig:
    vocab_size: int = 30522
    hidden_size: int = 1024
    num_layers: int = 24
    num_heads: int = 16
    intermediate_size: int = 4096
    max_position: int = 512
    type_vocab_size: int = 2
    dropout: float = 0.1
    layer_norm_eps: float = 1e-12
    # norm1 / norm2 of every layer as DropoutAddLayerNorm: the dropout, residual add and LayerNorm of each junction
    # run as one fused kernel per direction on CUDA (same parameters and state_dict as the stock layers)
    fused_norm: bool = False
    # the MLM loss through ops.xent.softmax_cross_entropy: one fused kernel per direction on CUDA reads the
    # low-precision logits in place of the fp32 cast and log-softmax of F.cross_entropy (same value)
    fused_loss: bool = False
    # qkv, proj, fc1 and fc2 of every encoder layer as ops.fp8.Fp8Linear: FP8 GEMMs with delayed scaling on sm_90
    # (same parameters and state_dict as nn.Linear); the heads stay in the model's dtype.  The GELU between fc1 and
    # fc2 then runs inside the FP8 casts (ops.fp8.fp8_gelu_mlp), with the same results
    fp8_linear: bool = False
    # self-attention through ops.attn.self_attention: one fused kernel forward and two backward on CUDA read Q, K and
    # V in place from the qkv projection and write the context and d(qkv) in the layouts the linears use (same
    # parameters and state_dict; other inputs run the stock SDPA expression)
    fused_attention: bool = False
    # k > 0: with mlm_labels, the MLM head (dense, GELU, LayerNorm, tied decoder, loss) runs on the first C = B k
    # labelled tokens of the batch only, gathered on the device by ops.mlm.gather_labelled, rather than on every token.
    # Labelled tokens past C take no loss and are counted in mlm_dropped_targets.  0: the head runs on every token
    max_predictions_per_seq: int = 0


class BertEmbeddings(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.word = nn.Embedding(c.vocab_size, c.hidden_size)
        self.pos = nn.Embedding(c.max_position, c.hidden_size)
        self.token_type = nn.Embedding(c.type_vocab_size, c.hidden_size)
        self.norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.drop = nn.Dropout(c.dropout)

    def forward(self, ids, type_ids, pos=None):
        if pos is None:
            pos = torch.arange(ids.shape[1], device=ids.device).unsqueeze(0)
        return self.drop(self.norm(self.word(ids) + self.pos(pos) + self.token_type(type_ids)))


def _junction_norm(c: BertConfig) -> nn.LayerNorm:
    if c.fused_norm:
        return DropoutAddLayerNorm(c.hidden_size, eps=c.layer_norm_eps, p=c.dropout)
    return nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)


def _encoder_linear(c: BertConfig, i: int, o: int) -> nn.Linear:
    return Fp8Linear(i, o) if c.fp8_linear else nn.Linear(i, o)


class BertLayer(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.h, self.d = c.num_heads, c.hidden_size // c.num_heads
        self.qkv = _encoder_linear(c, c.hidden_size, 3 * c.hidden_size)
        self.proj = _encoder_linear(c, c.hidden_size, c.hidden_size)
        self.norm1 = _junction_norm(c)
        self.fc1 = _encoder_linear(c, c.hidden_size, c.intermediate_size)
        self.fc2 = _encoder_linear(c, c.intermediate_size, c.hidden_size)
        self.norm2 = _junction_norm(c)
        self.p = c.dropout
        self.fused_norm = c.fused_norm
        self.fused_attention = c.fused_attention

    def forward(self, x, mask=None, cu_seqlens=None, max_seqlen=None):
        b, s, e = x.shape
        if self.fused_attention:
            a = self_attention(self.qkv(x), self.h, mask, self.p, self.training, cu_seqlens=cu_seqlens,
                               max_seqlen=max_seqlen)
        elif cu_seqlens is not None:
            a = _stock_varlen(self.qkv(x), self.h, cu_seqlens, max_seqlen, self.p if self.training else 0.0)
        else:
            q, k, v = self.qkv(x).view(b, s, 3, self.h, self.d).permute(2, 0, 3, 1, 4)
            a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=self.p if self.training else 0.0)
            a = a.transpose(1, 2).reshape(b, s, e)
        if self.fused_norm:
            x = self.norm1(self.proj(a), x)
            return self.norm2(self.mlp(x), x)
        x = self.norm1(x + F.dropout(self.proj(a), self.p, self.training))
        return self.norm2(x + F.dropout(self.mlp(x), self.p, self.training))

    def mlp(self, x):
        if isinstance(self.fc1, Fp8Linear):
            return fp8_gelu_mlp(x, self.fc1, self.fc2)
        return self.fc2(F.gelu(self.fc1(x)))


class BertForPreTraining(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.config = c
        self.embeddings = BertEmbeddings(c)
        self.layers = nn.ModuleList([BertLayer(c) for _ in range(c.num_layers)])
        self.pooler = nn.Linear(c.hidden_size, c.hidden_size)
        self.mlm_dense = nn.Linear(c.hidden_size, c.hidden_size)
        self.mlm_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.mlm_bias = nn.Parameter(torch.zeros(c.vocab_size))
        self.nsp = nn.Linear(c.hidden_size, 2)
        # labelled tokens that found no slot of the max_predictions_per_seq head, summed over every forward
        self.register_buffer("mlm_dropped_targets", torch.zeros((), dtype=torch.int64), persistent=False)
        self.apply(self._init)

    @staticmethod
    def _init(m):
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)

    def forward(self, ids, type_ids=None, mask=None, mlm_labels=None, nsp_labels=None, cu_seqlens=None,
                max_seqlen=None):
        """With ``cu_seqlens`` (device int32 [N + 1]), ``ids`` / ``type_ids`` / ``mlm_labels`` [B, S] are one packed
        stream of T = B S tokens read row-major, in which sequence n is tokens [cu[n], cu[n + 1]); ``mask`` must be
        None.  Token t takes position t - cu[n], NSP pools the first token of each sequence (``nsp_labels`` [N], -100
        for empty slots), tokens outside every sequence take no MLM loss, and attention stays inside each sequence.
        ``max_seqlen`` (default min(S, max_position)) bounds every length.  Nothing here reads cu_seqlens on the host,
        so a step with fixed shapes captures into one CUDA graph.

        With ``config.max_predictions_per_seq`` = k > 0 and ``mlm_labels``, the MLM head runs on the first B k
        labelled tokens in stream order only (in packed mode k counts per row of the B x S stream); the labelled
        tokens past them take no loss and are added to ``mlm_dropped_targets``."""
        if type_ids is None:
            type_ids = torch.zeros_like(ids)
        pos = first = None
        if cu_seqlens is not None:
            if mask is not None:
                raise ValueError("mask and cu_seqlens cannot be used together")
            b, s = ids.shape
            if max_seqlen is None:
                max_seqlen = min(s, self.config.max_position)
            t = torch.arange(b * s, device=ids.device)
            seq, inside = _packed_tokens(cu_seqlens, t)
            pos = (t - cu_seqlens[seq]).clamp(0, self.config.max_position - 1).view(b, s)
            first = cu_seqlens[:-1].clamp(0, b * s - 1).long()
            if mlm_labels is not None:
                mlm_labels = mlm_labels.masked_fill(~inside.view(b, s), -100)
        x = self.embeddings(ids, type_ids, pos)
        for layer in self.layers:
            x = layer(x, mask, cu_seqlens, max_seqlen)
        pooled = torch.tanh(self.pooler(x[:, 0] if first is None else x.reshape(-1, x.shape[-1])[first]))
        if mlm_labels is not None and self.config.max_predictions_per_seq > 0:
            x, mlm_labels, dropped = gather_labelled(x, mlm_labels, x.shape[0] * self.config.max_predictions_per_seq)
            self.mlm_dropped_targets.add_(dropped)
        h = self.mlm_norm(F.gelu(self.mlm_dense(x)))
        logits = F.linear(h, self.embeddings.word.weight, self.mlm_bias)   # tied decoder
        nsp_logits = self.nsp(pooled)
        if mlm_labels is None:
            return logits, nsp_logits
        if self.config.fused_loss:
            loss = softmax_cross_entropy(logits.view(-1, logits.shape[-1]), mlm_labels.view(-1), ignore_index=-100)
        else:
            loss = F.cross_entropy(logits.view(-1, logits.shape[-1]).float(), mlm_labels.view(-1), ignore_index=-100)
        if nsp_labels is not None:
            loss = loss + F.cross_entropy(nsp_logits.float(), nsp_labels)
        return loss


def bert_large(**kw):
    return BertForPreTraining(BertConfig(**kw))


def bert_base(**kw):
    cfg = dict(hidden_size=768, num_layers=12, num_heads=12, intermediate_size=3072)
    cfg.update(kw)
    return BertForPreTraining(BertConfig(**cfg))


def bert_tiny(**kw):
    """2-layer, 128-wide configuration for smoke tests and CPU runs of the examples."""
    cfg = dict(hidden_size=128, num_layers=2, num_heads=2, intermediate_size=512, max_position=128)
    cfg.update(kw)
    return BertForPreTraining(BertConfig(**cfg))


def num_params(model):
    return sum(p.numel() for p in model.parameters())


del math
