"""
Transformer (sup v5) model package -- host-side mirror of `bonito/transformer/model.py`.

The reference builds its layer from flash-attn modules (`RotaryEmbedding`, `GatedMlp`, Triton `RMSNorm`,
`flash_attn_qkvpacked_func`); here the same parameters (same `state_dict` names and shapes) sit in plain torch
modules whose `forward` spells out the arithmetic those kernels implement (flash-attn's own torch reference
functions: `rms_norm_ref`, `apply_rotary_emb_torch`, `swiglu_fwd`).  With `use_koi` armed the native engine
(`bonito_b200.engine_tf`) runs the stack on the sm_90a kernels instead.
"""

import types
from functools import lru_cache

import torch
import torch.nn.functional as F

from bonito_b200.crf.model import SeqdistModel  # noqa: F401  (registers `seqdistmodel`)
from bonito_b200.nn import from_dict, register, LinearCRFEncoder, MakeContiguous, Module, Permute, Serial


def deepnorm_params(depth):
    """DeepNorm (arXiv:2203.00555) alpha / beta for an encoder of `depth` layers."""
    return round((2 * depth) ** 0.25, 7), round((8 * depth) ** (-1 / 4), 7)


@lru_cache(maxsize=2)
def sliding_window_mask(seq_len, window, device):
    """True where query i may attend key j: i - window[0] <= j <= i + window[1]."""
    i = torch.arange(seq_len)[:, None]
    j = torch.arange(seq_len)[None, :]
    return ((j >= i - window[0]) & (j <= i + window[1])).to(device)


class RMSNorm(Module):
    """out = rmsnorm(x + residual) * weight, statistics in fp32, one rounding on store (eps 1e-5)."""

    def __init__(self, hidden_size, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.weight = torch.nn.Parameter(torch.ones(hidden_size))

    def forward(self, x, residual=None):
        dtype = x.dtype
        s = x.float() if residual is None else x.float() + residual.float()
        rstd = torch.rsqrt(s.square().mean(dim=-1, keepdim=True) + self.eps)
        return (s * rstd * self.weight.float()).to(dtype)


class GatedMlp(Module):
    """fc1 -> (y, gate) -> y * silu(gate) -> fc2 (SwiGLU; product formed in fp32, rounded once)."""

    def __init__(self, in_features, hidden_features, bias1=False, bias2=False):
        super().__init__()
        self.fc1 = torch.nn.Linear(in_features, 2 * hidden_features, bias=bias1)
        self.fc2 = torch.nn.Linear(hidden_features, in_features, bias=bias2)

    def forward(self, x):
        y, gate = self.fc1(x).chunk(2, dim=-1)
        g = gate.float()
        return self.fc2((g * y.float() / (1.0 + torch.exp(-g))).to(x.dtype))


def rotary_tables(seq_len, dim, dtype, device, base=10000.0):
    """cos / sin [seq_len, dim/2]: computed in fp32, then cast to the activations' dtype (flash-attn RotaryEmbedding)."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2, device=device, dtype=torch.float32) / dim))
    freqs = torch.outer(torch.arange(seq_len, device=device, dtype=torch.float32), inv_freq)
    return torch.cos(freqs).to(dtype), torch.sin(freqs).to(dtype)


def apply_rotary(x, cos, sin):
    """NeoX (half-split) rotation of x [N, T, heads, dim] in fp32, rounded to x.dtype."""
    half = x.shape[-1] // 2
    x1, x2 = x[..., :half].float(), x[..., half:].float()
    c, s = cos[None, :, None, :].float(), sin[None, :, None, :].float()
    return torch.cat([x1 * c - x2 * s, x1 * s + x2 * c], dim=-1).to(x.dtype)


class MultiHeadAttention(Module):
    def __init__(self, d_model, nhead, qkv_bias=False, out_bias=True, rotary_dim=None, attn_window=None):
        super().__init__()
        assert d_model % nhead == 0, "d_model must be divisible by nhead"
        self.d_model, self.nhead = d_model, nhead
        self.head_dim = d_model // nhead
        self.rotary_dim = self.head_dim if rotary_dim is None else rotary_dim
        self.Wqkv = torch.nn.Linear(d_model, 3 * d_model, bias=qkv_bias)
        self.out_proj = torch.nn.Linear(d_model, d_model, bias=out_bias)
        self.attn_window = (-1, -1) if attn_window is None else tuple(attn_window)

    def forward(self, x):
        N, T, _ = x.shape
        qkv = self.Wqkv(x).view(N, T, 3, self.nhead, self.head_dim)
        cos, sin = rotary_tables(T, self.rotary_dim, qkv.dtype, qkv.device)
        q = apply_rotary(qkv[:, :, 0], cos, sin).permute(0, 2, 1, 3)
        k = apply_rotary(qkv[:, :, 1], cos, sin).permute(0, 2, 1, 3)
        v = qkv[:, :, 2].permute(0, 2, 1, 3)
        mask = None
        if self.attn_window != (-1, -1):
            mask = sliding_window_mask(T, self.attn_window, q.device)
        out = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        return self.out_proj(out.permute(0, 2, 1, 3).reshape(N, T, self.d_model))


@register
class TransformerEncoderLayer(Module):
    """Post-norm DeepNorm block: x = norm1(attn(x) + a*x); x = norm2(ff(x) + a*x)."""

    def __init__(self, d_model, nhead, dim_feedforward, deepnorm_alpha, deepnorm_beta, attn_window=None):
        super().__init__()
        self.kwargs = dict(d_model=d_model, nhead=nhead, dim_feedforward=dim_feedforward,
                           deepnorm_alpha=deepnorm_alpha, deepnorm_beta=deepnorm_beta, attn_window=attn_window)
        self.self_attn = MultiHeadAttention(d_model, nhead, qkv_bias=False, out_bias=True, attn_window=attn_window)
        self.ff = GatedMlp(d_model, dim_feedforward, bias1=False, bias2=False)
        self.norm1 = RMSNorm(d_model)
        self.norm2 = RMSNorm(d_model)
        self.register_buffer("deepnorm_alpha", torch.tensor(deepnorm_alpha))
        self.reset_parameters()

    def reset_parameters(self):
        beta, d = self.kwargs["deepnorm_beta"], self.kwargs["d_model"]
        xavier = torch.nn.init.xavier_normal_
        xavier(self.ff.fc1.weight, gain=beta)
        xavier(self.ff.fc2.weight, gain=beta)
        xavier(self.self_attn.out_proj.weight, gain=beta)
        xavier(self.self_attn.Wqkv.weight[2 * d:], gain=beta)
        xavier(self.self_attn.Wqkv.weight[:2 * d], gain=1)

    def forward(self, x):
        x = self.norm1(self.self_attn(x), self.deepnorm_alpha * x)
        return self.norm2(self.ff(x), self.deepnorm_alpha * x)

    def to_dict(self, include_weights=False):
        if include_weights:
            raise NotImplementedError
        return self.kwargs


def use_koi(self, **kwargs):
    """Native mode: scores without blank column, batch-first [N, T, C] (reference: transformer/model.py:136-146)."""
    def _no_blanks(m):
        if isinstance(m, LinearCRFEncoder):
            m.expand_blanks = False
    self.encoder.apply(_no_blanks)
    self.encoder = Serial([self.encoder, Permute([1, 0, 2]), MakeContiguous()])
    self._native = dict(kwargs)
    self._plan = None


def Model(config):
    """`config['model']` describes a `seqdistmodel` whose encoder is a NamedSerial (conv, transformer_encoder, ...)."""
    model_config = {k: v for k, v in config["model"].items() if k != "package"}
    model = from_dict(model_config)
    model.config = config
    model.use_koi = types.MethodType(use_koi, model)
    return model
