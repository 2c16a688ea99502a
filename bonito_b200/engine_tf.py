"""
Plan builder + executor for the transformer (sup v5) encoder:

    NamedSerial(conv = Serial[Convolution x5, Permute([0,2,1])], transformer_encoder = Stack[TransformerEncoderLayer x18],
                upsample = LinearUpsample(x2), crf = LinearCRFEncoder(scale=5, permute=[1,0,2]))

(`bonito/models/configs/dna_r10.4.1@v5.0.toml`, `bonito/transformer/model.py:82-154`).  Like the
reference's `use_koi` rewrite it returns scores batch-first, `[N, 2T', C]` fp16 without the blank column.

Schedule per batch: conv_first kernel (1->64), four convolutions as wgmma GEMMs over overlapping channels-last rows
(swish in the epilogue, output written straight into the next layer's zero-haloed buffer), then per layer
QKV GEMM -> rotary + windowed attention -> out-proj GEMM (+bias) -> residual RMSNorm -> fc1 GEMM -> SwiGLU -> fc2 GEMM ->
residual RMSNorm, then the upsample GEMM (+bias; the x2 reshape is free in a batch-first layout) and the CRF GEMM (x scale).
"""

import os

import torch

from bonito_b200 import native
from bonito_b200 import nn as bnn
from bonito_b200.engine import UnsupportedModel, _Stage, _act_code, _dev16, _folded_conv

# SwiGLU formed in the fc1 GEMM's epilogue (B200_ACT_SWIGLU); B200_FUSE_SWIGLU=0 keeps the separate kernel as a cross-check
FUSE_SWIGLU = os.environ.get("B200_FUSE_SWIGLU", "1") != "0"


def _interleave_swiglu(w1):
    """fc1.weight [2F, d] (rows: y then gate, GatedMlp's chunk(2)) -> rows in 64-groups [32 y | 32 gate] of the same features."""
    f = w1.shape[0] // 2
    assert f % 32 == 0, "fused SwiGLU needs dim_feedforward % 32 == 0"
    y, g = w1[:f].reshape(f // 32, 32, -1), w1[f:].reshape(f // 32, 32, -1)
    return torch.cat([y, g], dim=1).reshape(2 * f, -1).contiguous()


def find_transformer_encoder(encoder):
    """The NamedSerial(conv, transformer_encoder, upsample, crf) inside an encoder (possibly wrapped by use_koi)."""
    for m in encoder.modules():
        if isinstance(m, bnn.NamedSerial) and hasattr(m, "transformer_encoder"):
            return m
    return None


class TransformerPlan:
    supports_slots = True      # buffers are keyed by (N, L, slot)

    def __init__(self, encoder, device):
        from bonito_b200.transformer.model import TransformerEncoderLayer
        enc = find_transformer_encoder(encoder)
        if enc is None:
            raise UnsupportedModel("no conv / transformer_encoder / upsample / crf stack found")
        self.device = dev = torch.device(device)
        convs = [m for m in enc.conv.children() if isinstance(m, bnn.Convolution)]
        if len(convs) < 2 or convs[0].conv.in_channels != 1:
            raise UnsupportedModel("transformer conv stack must start from a single input feature")
        self.convs = []
        for i, c in enumerate(convs):
            w, b = _folded_conv(c)
            cout, cin, k = w.shape
            s, p = c.conv.stride[0], c.conv.padding[0]
            if i == 0:
                if s != 1 or p != k // 2:
                    raise UnsupportedModel("first convolution must be stride 1 with 'same' padding")
                wp = _dev16(w, dev)
            else:
                wp = _dev16(w.permute(0, 2, 1).reshape(cout, -1), dev)   # [Cout][tap*Cin + cin]
                if (k * cin) % 8 or (s * cin) % 8 or cout % 8:
                    raise UnsupportedModel("convolution widths must be multiples of 8")
            self.convs.append(dict(w=wp, b=_dev16(b, dev), cin=cin, cout=cout, k=k, s=s, p=p, act=_act_code(c.activation)))

        self.layers = []
        for layer in enc.transformer_encoder:
            if not isinstance(layer, TransformerEncoderLayer):
                raise UnsupportedModel(f"unsupported layer {type(layer).__name__} in transformer_encoder")
            a = layer.self_attn
            if a.head_dim != 64 or a.rotary_dim != 64 or a.Wqkv.bias is not None:
                raise UnsupportedModel("native attention needs head_dim = rotary_dim = 64 and no qkv bias")
            self.layers.append(dict(
                wqkv=_dev16(a.Wqkv.weight.detach(), dev),
                wo=_dev16(a.out_proj.weight.detach(), dev),
                bo=_dev16(None if a.out_proj.bias is None else a.out_proj.bias.detach(), dev),
                w1=_dev16(_interleave_swiglu(layer.ff.fc1.weight.detach()), dev) if FUSE_SWIGLU else
                _dev16(layer.ff.fc1.weight.detach(), dev),
                w2=_dev16(layer.ff.fc2.weight.detach(), dev),
                n1=_dev16(layer.norm1.weight.detach(), dev), n2=_dev16(layer.norm2.weight.detach(), dev),
                eps=float(layer.norm1.eps),
                # deepnorm_alpha is a buffer that model.half() rounds to fp16 (2.4494897 -> 2.4492188)
                alpha=float(layer.deepnorm_alpha.detach().to(torch.float16).float()),
                window=tuple(a.attn_window), nhead=a.nhead))
        self.d_model = enc.transformer_encoder[0].self_attn.d_model
        self.d_ff = enc.transformer_encoder[0].ff.fc2.in_features

        up = enc.upsample
        if not up.batch_first:
            raise UnsupportedModel("native LinearUpsample needs batch_first=True")
        self.up_factor = up.scale_factor
        self.wu, self.bu = _dev16(up.linear.weight.detach(), dev), _dev16(up.linear.bias.detach(), dev)
        crf = enc.crf
        if crf.activation is not None or crf.blank_score is None or crf.linear.bias is not None:
            raise UnsupportedModel("native CRF head supports activation=None, bias=False and a fixed blank_score")
        self.wc = _dev16(crf.linear.weight.detach(), dev)
        self.scale = None if crf.scale is None else float(crf.scale)
        self.state_len, self.blank_score, self.n_scores = crf.state_len, float(crf.blank_score), self.wc.shape[0]
        self._bufs = {}

    # ------------------------------------------------------------------------------------------------
    def _geometry(self, L):
        """Per conv: input length, output length, padded row count of the INPUT buffer (multiple of the stride)."""
        geo, lin = [], L
        for c in self.convs:
            lout = (lin + 2 * c["p"] - c["k"]) // c["s"] + 1
            need = max(c["p"] + lin, (lout - 1) * c["s"] + c["k"])
            rows = -(-need // c["s"]) * c["s"]
            geo.append(dict(lin=lin, lout=lout, lp=rows))
            lin = lout
        return geo

    def frames(self, L):
        return self._geometry(L)[-1]["lout"] * self.up_factor

    def _buffers(self, N, L, slot=0):
        key = (N, L, slot)
        if key not in self._bufs:
            for k in [k for k in self._bufs if k[:2] != (N, L)]:
                del self._bufs[k]
            geo = self._geometry(L)
            dev, f16 = self.device, torch.float16
            bufs = dict(geo=geo, act=[])
            # act[i] = input buffer of conv i+1 (output of conv i), channels-last with zero halo; i = 0 .. n-2
            for i in range(len(self.convs) - 1):
                nxt, c = self.convs[i + 1], self.convs[i]
                lp = geo[i + 1]["lp"]
                t = torch.zeros(N * lp * c["cout"] + nxt["k"] * nxt["cin"], dtype=f16, device=dev)
                bufs["act"].append(t)
            Tq = geo[-1]["lout"]
            M, d, ff = N * Tq, self.d_model, self.d_ff
            bufs.update(T=Tq, M=M,
                        xa=torch.empty(M, d, dtype=f16, device=dev), xb=torch.empty(M, d, dtype=f16, device=dev),
                        qkv=torch.empty(M, 3 * d, dtype=f16, device=dev), att=torch.empty(M, d, dtype=f16, device=dev),
                        proj=torch.empty(M, d, dtype=f16, device=dev), h1=None if FUSE_SWIGLU else torch.empty(M, 2 * ff, dtype=f16, device=dev),
                        g=torch.empty(M, ff, dtype=f16, device=dev),
                        up=torch.empty(M, self.up_factor * d, dtype=f16, device=dev))
            inv_freq = 1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float32, device=dev) / 64))
            freqs = torch.outer(torch.arange(Tq, dtype=torch.float32, device=dev), inv_freq)
            bufs["cos_sin"] = torch.cat([torch.cos(freqs), torch.sin(freqs)], dim=1).to(f16).contiguous()
            self._bufs[key] = bufs
        return self._bufs[key]

    def forward(self, x, out=None, events=None, return_features=False, slot=0, **_):
        with torch.cuda.device(self.device):    # streams / events / launches belong to the plan's device, whatever is current
            return self._forward(x, out=out, events=events, return_features=return_features, slot=slot)

    def _forward(self, x, out=None, events=None, return_features=False, slot=0):
        if x.dim() == 3:
            x = x[:, 0, :]
        x = x.to(device=self.device, dtype=torch.float16).contiguous()
        N, L = x.shape
        b = self._buffers(N, L, slot)
        geo, T, M, d, ff = b["geo"], b["T"], b["M"], self.d_model, self.d_ff
        feats = {}

        def stage(name):
            return _Stage(name, events)

        c0 = self.convs[0]
        with stage("conv_first"):
            native.conv_first(x, c0["w"], c0["b"], c0["act"], b["act"][0], geo[1]["lp"], self.convs[1]["p"])
        for i in range(1, len(self.convs)):
            c, g = self.convs[i], geo[i]
            src = b["act"][i - 1]
            rows = g["lp"] // c["s"]
            if i + 1 < len(self.convs):   # into the next conv's haloed buffer: row (n, t) -> n * lp_next + pad_next + t
                dst = b["act"][i][self.convs[i + 1]["p"] * c["cout"]:]
                so = geo[i + 1]["lp"]
            else:                          # last conv: the transformer input x [N, T, d]
                dst, so = b["xa"], g["lout"]
            with stage("conv_gemm"):
                native.gemm(src, c["s"] * c["cin"], c["w"], c["b"], dst, c["cout"], N * rows, c["cout"], c["k"] * c["cin"],
                            act=c["act"], rows_inner=rows, valid_inner=g["lout"], stride_inner=1, stride_outer=so)
        cur, nxt = b["xa"], b["xb"]
        if return_features:
            feats["conv"] = cur.view(N, T, d).clone()

        for li, l in enumerate(self.layers):
            with stage("qkv_gemm"):
                native.gemm(cur, d, l["wqkv"], None, b["qkv"], 3 * d, M, 3 * d, d)
            with stage("attention"):
                native.attention(b["qkv"], b["cos_sin"], b["att"], N, T, l["nhead"], 64, l["window"][0], l["window"][1])
            with stage("proj_gemm"):
                native.gemm(b["att"], d, l["wo"], l["bo"], b["proj"], d, M, d, d)
            with stage("rmsnorm"):
                native.rmsnorm_residual(b["proj"], cur, l["n1"], l["alpha"], l["eps"], nxt, M, d)
            cur, nxt = nxt, cur
            if FUSE_SWIGLU:
                with stage("fc1_swiglu_gemm"):   # y * silu(gate) formed in the GEMM epilogue: h1 never reaches HBM
                    native.gemm(cur, d, l["w1"], None, b["g"], ff, M, 2 * ff, d, act=native.ACT_SWIGLU)
            else:
                with stage("fc1_gemm"):
                    native.gemm(cur, d, l["w1"], None, b["h1"], 2 * ff, M, 2 * ff, d)
                with stage("swiglu"):
                    native.swiglu(b["h1"], b["g"], M, ff)
            with stage("fc2_gemm"):
                native.gemm(b["g"], ff, l["w2"], None, b["proj"], d, M, d, ff)
            with stage("rmsnorm"):
                native.rmsnorm_residual(b["proj"], cur, l["n2"], l["alpha"], l["eps"], nxt, M, d)
            cur, nxt = nxt, cur
            if return_features:
                feats[f"layer{li}"] = cur.view(N, T, d).clone()

        with stage("upsample_gemm"):
            native.gemm(cur, d, self.wu, self.bu, b["up"], self.up_factor * d, M, self.up_factor * d, d)
        Mu = M * self.up_factor                         # [N, T, f*d] viewed as [N, f*T, d]: same memory
        if out is None:
            out = torch.empty(N, T * self.up_factor, self.n_scores, dtype=torch.float16, device=self.device)
        with stage("crf_gemm"):
            native.gemm(b["up"], d, self.wc, None, out, self.n_scores, Mu, self.n_scores, d,
                        act=native.ACT_NONE if self.scale is None else native.ACT_SCALE, lo=self.scale or 0.0)
        return (out, feats) if return_features else out


def compile_transformer(encoder, device):
    return TransformerPlan(encoder, device)
