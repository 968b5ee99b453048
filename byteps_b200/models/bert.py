"""BERT encoder with the pre-training heads (MLM + NSP): the reference's
bandwidth-bound headline workload (BERT-large, ~335 M parameters,
/root/reference/README.md:36-38)."""
import math
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.attn import self_attention
from ..ops.fp8 import Fp8Linear, fp8_gelu_mlp
from ..ops.ln import DropoutAddLayerNorm
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


class BertEmbeddings(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.word = nn.Embedding(c.vocab_size, c.hidden_size)
        self.pos = nn.Embedding(c.max_position, c.hidden_size)
        self.token_type = nn.Embedding(c.type_vocab_size, c.hidden_size)
        self.norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.drop = nn.Dropout(c.dropout)

    def forward(self, ids, type_ids):
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

    def forward(self, x, mask=None):
        b, s, e = x.shape
        if self.fused_attention:
            a = self_attention(self.qkv(x), self.h, mask, self.p, self.training)
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
        self.apply(self._init)

    @staticmethod
    def _init(m):
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)

    def forward(self, ids, type_ids=None, mask=None, mlm_labels=None, nsp_labels=None):
        if type_ids is None:
            type_ids = torch.zeros_like(ids)
        x = self.embeddings(ids, type_ids)
        for layer in self.layers:
            x = layer(x, mask)
        pooled = torch.tanh(self.pooler(x[:, 0]))
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
