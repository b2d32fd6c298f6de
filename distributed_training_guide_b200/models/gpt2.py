"""GPT-2 (LayerNorm, learned positions, GELU-new, Conv1D+bias, tied head, dropout).

This is the model of the guide's smoke command (``-m openai-community/gpt2``, reference
``01-single-gpu/README.md:9-12``) and of BASELINE.json's config 01, which is a CPU
plumbing configuration.  It is therefore written in plain PyTorch ops (SURVEY.md K4b);
the sm_90a kernels target the Llama family.  Parameter names follow HF's
``GPT2LMHeadModel`` (``transformer.wte.weight`` ... ``transformer.h.{i}.attn.c_attn.weight``).
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch
import torch.utils.checkpoint
import torch.nn.functional as F
from torch import nn

from ..ops import reference as ref
from .configs import ModelConfig


class Conv1D(nn.Module):
    """HF's GPT-2 'Conv1D': a linear layer whose weight is stored [in, out]."""

    def __init__(self, nin, nout, dtype=None, device=None):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(nin, nout, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(nout, dtype=dtype, device=device))

    def forward(self, x):
        return torch.addmm(self.bias, x.reshape(-1, x.shape[-1]), self.weight).view(*x.shape[:-1], -1)


class GPT2Attention(nn.Module):
    def __init__(self, cfg, dtype, device):
        super().__init__()
        self.nh = cfg.num_attention_heads
        self.c_attn = Conv1D(cfg.hidden_size, 3 * cfg.hidden_size, dtype, device)
        self.c_proj = Conv1D(cfg.hidden_size, cfg.hidden_size, dtype, device)
        self.p = cfg.dropout

    def forward(self, x):
        B, S, H = x.shape
        q, k, v = self.c_attn(x).view(B, S, 3, self.nh, H // self.nh).unbind(2)
        o = F.scaled_dot_product_attention(
            q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True,
            dropout_p=self.p if self.training else 0.0,
        )
        o = o.transpose(1, 2).reshape(B, S, H)
        return F.dropout(self.c_proj(o), self.p, self.training)


class GPT2MLP(nn.Module):
    def __init__(self, cfg, dtype, device):
        super().__init__()
        self.c_fc = Conv1D(cfg.hidden_size, cfg.intermediate_size, dtype, device)
        self.c_proj = Conv1D(cfg.intermediate_size, cfg.hidden_size, dtype, device)
        self.p = cfg.dropout

    def forward(self, x):
        return F.dropout(self.c_proj(ref.gelu_new(self.c_fc(x))), self.p, self.training)


class GPT2Block(nn.Module):
    def __init__(self, cfg, dtype, device):
        super().__init__()
        self.ln_1 = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_epsilon, dtype=dtype, device=device)
        self.attn = GPT2Attention(cfg, dtype, device)
        self.ln_2 = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_epsilon, dtype=dtype, device=device)
        self.mlp = GPT2MLP(cfg, dtype, device)

    def forward(self, x):
        x = x + self.attn(self.ln_1(x))
        return x + self.mlp(self.ln_2(x))


class GPT2Model(nn.Module):
    def __init__(self, cfg, dtype, device):
        super().__init__()
        self.wte = nn.Embedding(cfg.vocab_size, cfg.hidden_size, dtype=dtype, device=device)
        self.wpe = nn.Embedding(cfg.max_position_embeddings, cfg.hidden_size, dtype=dtype, device=device)
        self.h = nn.ModuleList([GPT2Block(cfg, dtype, device) for _ in range(cfg.num_hidden_layers)])
        self.ln_f = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_epsilon, dtype=dtype, device=device)
        self.p = cfg.dropout

    @property
    def layers(self):  # uniform access for the parallel engines (model.model.layers)
        return self.h


@torch.no_grad()
def init_parameter_(p, name: str, seed: int, n_layer: int, std: float = 0.02):
    """GPT-2 initialisation of one parameter as a pure function of (seed, name): biases 0, LayerNorm gains 1, residual
    projections N(0, std / sqrt(2 L)), everything else N(0, std) — the same values under every parallel layout (the
    sharded engine materialises one group at a time and keeps only its slice)."""
    from .llama import _name_seed

    if name.endswith("bias"):
        p.zero_()
    elif "ln_" in name:
        p.fill_(1.0)
    else:
        s = std / math.sqrt(2 * n_layer) if name.endswith("c_proj.weight") else std
        gen = torch.Generator(device=p.device)
        gen.manual_seed(_name_seed(seed, name))
        p.copy_(torch.empty(tuple(p.shape), dtype=torch.float32, device=p.device).normal_(0.0, s, generator=gen).to(p.dtype))


class GPT2LMHeadModel(nn.Module):
    def __init__(self, config: ModelConfig, dtype=None, device=None):
        super().__init__()
        self.config = config
        self.transformer = GPT2Model(config, dtype, device)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False, dtype=dtype, device=device)
        self.lm_head.weight = self.transformer.wte.weight  # tied
        #: parallel engine (parallel/ddp.py): the same hook protocol as the Llama model — called around every block
        #: and in front of the head so that gradient buckets are reduced as soon as they are final
        self.engine = None
        self.activation_checkpointing = False

    @property
    def model(self):
        return self.transformer

    @torch.no_grad()
    def init_weights(self, std=0.02, seed=0):
        n_layer = self.config.num_hidden_layers
        seen = set()
        for name, p in self.named_parameters():
            if p.is_meta or id(p) in seen:
                continue
            seen.add(id(p))
            init_parameter_(p, name, seed, n_layer, std)

    def num_parameters(self):
        return sum(p.numel() for p in self.parameters())

    @staticmethod
    def loss_function(logits, labels, vocab_size=None):
        return ref.cross_entropy(logits.reshape(-1, logits.shape[-1]), ref.shift_labels(labels).reshape(-1))

    def forward(self, input_ids, attention_mask=None, labels=None, position_ids=None, return_logits=True):
        B, S = input_ids.shape
        t = self.transformer
        if position_ids is None:
            position_ids = torch.arange(S, device=input_ids.device)
        eng = self.engine
        if eng is not None:
            eng.pre_forward(self)
        x = t.wte(input_ids) + t.wpe(position_ids)
        x = F.dropout(x, t.p, self.training)
        for i, blk in enumerate(t.h):
            if eng is not None:
                x, _ = eng.pre_layer(i, blk, x, None)
            if self.activation_checkpointing and torch.is_grad_enabled():
                # --checkpoint-activations: keep only the block input, re-run the block in backward (the
                # RNG state is restored for the replay, so dropout masks match)
                x = torch.utils.checkpoint.checkpoint(blk, x, use_reentrant=False)
            else:
                x = blk(x)
            if eng is not None:
                x, _ = eng.post_layer(i, blk, x, None)
        if eng is not None:
            x, _ = eng.pre_head(x, None)
        logits = self.lm_head(t.ln_f(x))
        loss = self.loss_function(logits, labels) if labels is not None else None
        return SimpleNamespace(loss=loss, logits=logits)
