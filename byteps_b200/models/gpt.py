"""GPT-2-style decoder-only language model (pre-LN blocks, causal self-attention, LM head tied to the token
embedding), trained on next-token prediction over padded batches or packed variable-length streams."""
import math
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.attn import _packed_tokens, _stock, _stock_varlen, self_attention
from ..ops.fp8 import Fp8Linear, fp8_gelu_mlp
from ..ops.ln import DropoutAddLayerNorm
from ..ops.xent import softmax_cross_entropy


@dataclass
class GptConfig:
    # GPT-2's 50257 tokens padded to a multiple of 64, so every logits row starts on a 16-byte boundary
    vocab_size: int = 50304
    hidden_size: int = 768
    num_layers: int = 12
    num_heads: int = 12
    intermediate_size: int = 3072
    max_position: int = 1024
    dropout: float = 0.1
    layer_norm_eps: float = 1e-5
    # causal self-attention through ops.attn.self_attention(causal=True): one fused kernel forward and two backward
    # on CUDA that skip the key tiles above the diagonal (same parameters and state_dict; other inputs run the stock
    # SDPA expression)
    fused_attention: bool = False
    # the LM loss through ops.xent.softmax_cross_entropy: one fused kernel per direction on CUDA reads the
    # low-precision logits in place of the fp32 cast and log-softmax of F.cross_entropy (same value)
    fused_loss: bool = False
    # qkv, proj, fc1 and fc2 of every block as ops.fp8.Fp8Linear with the GELU inside the FP8 casts
    # (ops.fp8.fp8_gelu_mlp); same parameters and state_dict as nn.Linear.  The LM head stays in the model's dtype
    fp8_linear: bool = False
    # every LayerNorm (ln1, ln2, ln_f) as ops.ln.DropoutAddLayerNorm, run with the dropout and residual add in front
    # of it and returning their sum as the residual stream: one fused kernel per direction on CUDA at each of the
    # 2 L + 1 junctions (same parameters and state_dict; other inputs run the stock composition)
    fused_norm: bool = False


def _block_linear(c: GptConfig, i: int, o: int) -> nn.Linear:
    return Fp8Linear(i, o) if c.fp8_linear else nn.Linear(i, o)


def _norm(c: GptConfig) -> nn.LayerNorm:
    if c.fused_norm:
        return DropoutAddLayerNorm(c.hidden_size, eps=c.layer_norm_eps, p=c.dropout)
    return nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)


class GptBlock(nn.Module):
    """x + drop(proj(attn(ln1(x)))), then x + drop(mlp(ln2(x))).  With fused_norm the model runs the block
    through fused_forward instead, where each LayerNorm also forms the residual sum in front of it."""

    def __init__(self, c: GptConfig):
        super().__init__()
        self.h = c.num_heads
        self.ln1 = _norm(c)
        self.qkv = _block_linear(c, c.hidden_size, 3 * c.hidden_size)
        self.proj = _block_linear(c, c.hidden_size, c.hidden_size)
        self.ln2 = _norm(c)
        self.fc1 = _block_linear(c, c.hidden_size, c.intermediate_size)
        self.fc2 = _block_linear(c, c.intermediate_size, c.hidden_size)
        self.p = c.dropout
        self.fused_attention = c.fused_attention
        self.fused_norm = c.fused_norm

    def forward(self, x, cu_seqlens=None, max_seqlen=None):
        if self.fused_norm:
            raise RuntimeError("a fused_norm block runs through fused_forward")
        a = self.attn(self.qkv(self.ln1(x)), cu_seqlens, max_seqlen)
        x = x + F.dropout(self.proj(a), self.p, self.training)
        return x + F.dropout(self.mlp(self.ln2(x)), self.p, self.training)

    def fused_forward(self, x, a, next_ln, cu_seqlens=None, max_seqlen=None):
        """(x, a = ln1(x)) -> (next_ln(x'), x') for the block's output x', where next_ln is the next block's ln1
        or the final ln_f: each LayerNorm takes the dropout and residual add in front of it and returns the sum."""
        b, h = self.ln2(self.proj(self.attn(self.qkv(a), cu_seqlens, max_seqlen)), residual=x, return_sum=True)
        return next_ln(self.mlp(b), residual=h, return_sum=True)

    def attn(self, qkv, cu_seqlens, max_seqlen):
        if self.fused_attention:
            return self_attention(qkv, self.h, None, self.p, self.training, cu_seqlens=cu_seqlens,
                                  max_seqlen=max_seqlen, causal=True)
        p = self.p if self.training else 0.0
        if cu_seqlens is not None:
            return _stock_varlen(qkv, self.h, cu_seqlens, max_seqlen, p, causal=True)
        return _stock(qkv, self.h, None, p, causal=True)

    def mlp(self, x):
        if isinstance(self.fc1, Fp8Linear):
            return fp8_gelu_mlp(x, self.fc1, self.fc2)
        return self.fc2(F.gelu(self.fc1(x)))


class GptLMHeadModel(nn.Module):
    def __init__(self, c: GptConfig):
        super().__init__()
        self.config = c
        self.wte = nn.Embedding(c.vocab_size, c.hidden_size)
        self.wpe = nn.Embedding(c.max_position, c.hidden_size)
        self.blocks = nn.ModuleList([GptBlock(c) for _ in range(c.num_layers)])
        self.ln_f = _norm(c)
        self.apply(self._init)
        # GPT-2 scales the projections that feed the residual stream by 1 / sqrt(2 L)
        for blk in self.blocks:
            for lin in (blk.proj, blk.fc2):
                nn.init.normal_(lin.weight, std=0.02 / math.sqrt(2 * c.num_layers))

    @staticmethod
    def _init(m):
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)

    def forward(self, ids, labels=None, cu_seqlens=None, max_seqlen=None):
        """Next-token loss of ``ids`` [B, S] when ``labels`` is given, else the logits [B, S, V].

        ``labels`` is aligned with ``ids`` (as in Hugging Face): position t is trained on labels[t + 1], and -100
        takes no loss, so a padded batch marks its pads with -100 and needs no attention mask.  With ``cu_seqlens``
        (device int32 [N + 1]) ``ids`` / ``labels`` are one packed stream of T = B S tokens read row-major, in which
        sequence n is tokens [cu[n], cu[n + 1]): token t takes position t - cu[n], attention stays inside each
        sequence, and a target that crosses a sequence boundary or lies outside every sequence is ignored.
        ``max_seqlen`` (default min(S, max_position)) bounds every length.  Nothing here reads cu_seqlens on the
        host, so a step with fixed shapes captures into one CUDA graph."""
        b, s = ids.shape
        if cu_seqlens is not None:
            if max_seqlen is None:
                max_seqlen = min(s, self.config.max_position)
            t = torch.arange(b * s, device=ids.device)
            seq, inside = _packed_tokens(cu_seqlens, t)
            pos = (t - cu_seqlens[seq]).clamp(0, self.config.max_position - 1).view(b, s)
        else:
            pos = torch.arange(s, device=ids.device).unsqueeze(0)
        e = self.wte(ids) + self.wpe(pos)
        if self.config.fused_norm:
            # the embedding dropout runs inside the first ln1, each block's last residual add inside the next ln1
            a, x = self.blocks[0].ln1(e, return_sum=True)
            for i, blk in enumerate(self.blocks):
                next_ln = self.blocks[i + 1].ln1 if i + 1 < len(self.blocks) else self.ln_f
                a, x = blk.fused_forward(x, a, next_ln, cu_seqlens, max_seqlen)
        else:
            x = F.dropout(e, self.config.dropout, self.training)
            for blk in self.blocks:
                x = blk(x, cu_seqlens, max_seqlen)
            a = self.ln_f(x)
        logits = F.linear(a, self.wte.weight)   # tied LM head
        if labels is None:
            return logits
        # shift the labels rather than the logits, so the [T, V] logits stay one contiguous tensor
        if cu_seqlens is None:
            target = F.pad(labels[:, 1:], (0, 1), value=-100).reshape(-1)
        else:
            flat = labels.reshape(-1)
            same = inside[:-1] & inside[1:] & (seq[:-1] == seq[1:])
            target = F.pad(flat[1:].masked_fill(~same, -100), (0, 1), value=-100)
        logits = logits.view(-1, logits.shape[-1])
        if self.config.fused_loss:
            return softmax_cross_entropy(logits, target, ignore_index=-100)
        # in fp32, or in the logits' dtype when that is wider
        wide = torch.promote_types(logits.dtype, torch.float32)
        return F.cross_entropy(logits.to(wide), target, ignore_index=-100)


def gpt_tiny(**kw):
    """2-layer, 128-wide configuration for smoke tests and CPU runs."""
    cfg = dict(hidden_size=128, num_layers=2, num_heads=2, intermediate_size=512, max_position=512)
    cfg.update(kw)
    return GptLMHeadModel(GptConfig(**cfg))


def gpt2_small(**kw):
    """GPT-2 small: 12 layers of 768, 124 M parameters."""
    return GptLMHeadModel(GptConfig(**kw))


def gpt2_medium(**kw):
    """GPT-2 medium: 24 layers of 1024, 350 M parameters."""
    cfg = dict(hidden_size=1024, num_layers=24, num_heads=16, intermediate_size=4096)
    cfg.update(kw)
    return GptLMHeadModel(GptConfig(**cfg))
