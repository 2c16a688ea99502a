"""
Plan builder + executor for the QuartzNet CTC models (`package = "bonito.ctc"`: dna_r9.4.1@v1, @v2;
`bonito/ctc/model.py`).

`CtcPlan(model)` walks the `Encoder` / `Block` / `TCSConv1d` / `Decoder` tree, folds every BatchNorm into the weights and
bias of the convolution in front of it (with the module's own eps and running statistics) and packs fp16 operands once.
Schedule per batch, all channels-last `[N * T][C]` rows:

  * C1 (1 -> C, stride 3, dense): `b200_conv_first_fwd_ex`, written straight into the next block's input columns;
  * a separable block: per repeat one depthwise launch (`b200_depthwise_conv_fwd`) and one pointwise GEMM
    (`b200_gemm_fwd_ex`, activation in the epilogue).  In a residual block the last pointwise conv and the residual 1x1
    conv are ONE GEMM over the concatenated operand `[depthwise out | block input]` with weights `[W_pw s1 | W_res s2]` and
    bias `b1 + b2`: the layer in front of the block writes its output into the right-hand columns of that buffer and the
    last depthwise launch the left-hand ones;
  * a dense block: one GEMM, over overlapping rows of a zero-haloed buffer when k > 1 (v2's C3, k15);
  * the head (`b200_ctc_head_fwd`): logits, log_softmax, per-frame argmax and its probability.

fp16 deviation from the reference's module-by-module rounding: the folded BatchNorm means a convolution and its BatchNorm
round once instead of twice, and the residual sum is formed before that one rounding.

`forward(x)` returns `[N, T, 5]` fp16 log-probs (batch-first, like the other native plans), `greedy(x)` the per-frame
labels (uint8) and probabilities (fp32) `[N, T]` without materialising the log-probs.  Buffers are cached per (N, L).
Anything outside the shape rules of the two configs raises `UnsupportedModel`.
"""

import torch

from bonito_b200 import native
from bonito_b200.engine import UnsupportedModel, _Stage, _dev16

_ACTS = {"relu": native.ACT_RELU, "swish": native.ACT_SWISH}
DEPTHWISE_TAPS = (5, 9, 31, 33, 39, 51, 63, 67, 75, 87, 115, 123)   # kernel sizes b200_depthwise_conv_fwd supports


def depthwise_supported(c, k):
    return 256 <= c <= 512 and c % 8 == 0 and k in DEPTHWISE_TAPS


def _fold(conv, bn):
    """(weight, bias) in float64 of a bias-free Conv1d followed by an eval-mode BatchNorm1d."""
    w = conv.weight.detach().double()
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    b = bn.bias.detach().double() - bn.running_mean.detach().double() * s
    if conv.bias is not None:
        b = b + conv.bias.detach().double() * s
    return w * s[:, None, None], b


class CtcPlan:
    supports_slots = False

    def __init__(self, model, device, quantize=False):
        from bonito_b200.ctc.model import Block, TCSConv1d
        if quantize:
            raise UnsupportedModel("int8 (--quantize) has no native path for the QuartzNet CTC models")
        self.device = dev = torch.device(device)
        blocks = list(model.encoder.encoder)
        if not blocks or not all(isinstance(b, Block) for b in blocks):
            raise UnsupportedModel("native CTC path needs an Encoder of Blocks")
        self.blocks = []
        for i, blk in enumerate(blocks):
            act = blk.activation[0]
            name = getattr(type(act), "name", None)
            if name not in _ACTS:
                raise UnsupportedModel(f"activation {act!r} has no native kernel (relu, swish)")
            mods = [m for m in blk.conv if isinstance(m, (TCSConv1d, torch.nn.BatchNorm1d))]
            pairs = list(zip(mods[0::2], mods[1::2]))
            if len(mods) % 2 or not all(isinstance(t, TCSConv1d) and isinstance(b, torch.nn.BatchNorm1d) for t, b in pairs):
                raise UnsupportedModel("a Block must be repeat x [TCSConv1d, BatchNorm1d]")
            separable = pairs[0][0].separable
            convs = [t.depthwise if separable else t.conv for t, _ in pairs]
            k = convs[0].kernel_size[0]
            for c in convs + ([t.pointwise for t, _ in pairs] if separable else []):
                if c.dilation[0] != 1:
                    raise UnsupportedModel("dilated convolutions have no native kernel")
                if c.padding[0] != c.kernel_size[0] // 2:
                    raise UnsupportedModel("convolutions must use padding k // 2")
            stride = convs[0].stride[0]
            if i == 0:
                if separable or convs[0].in_channels != 1 or len(pairs) != 1 or blk.use_res:
                    raise UnsupportedModel("the first block must be a 1-channel dense convolution with repeat 1")
                if stride > 8 or k > 33 or k % 2 == 0 or convs[0].out_channels > 512:
                    raise UnsupportedModel(f"first convolution 1 -> {convs[0].out_channels} k{k} s{stride} has no native kernel")
            elif stride != 1:
                raise UnsupportedModel("only the first block may be strided")
            elif k % 2 == 0:        # padding k // 2 would give T + 1 frames: every block here keeps T
                raise UnsupportedModel(f"an even kernel size (k{k}) has no native path")
            if not separable and blk.use_res:
                raise UnsupportedModel("a residual connection on a non-separable block has no native path")
            if not separable and len(pairs) > 1:
                raise UnsupportedModel("a non-separable block with repeat > 1 has no native path")
            act_code = _ACTS[name]
            cin = pairs[0][0].depthwise.in_channels if separable else convs[0].in_channels
            cout = pairs[-1][1].num_features
            b = dict(separable=separable, residual=bool(blk.use_res), act=act_code, k=k, stride=stride, cin=cin, cout=cout,
                     reps=[])
            if separable:
                for r, (t, bn) in enumerate(pairs):
                    cdw = t.depthwise.in_channels
                    if not depthwise_supported(cdw, k):
                        raise UnsupportedModel(f"depthwise convolution C={cdw} k{k} has no native kernel")
                    w, bias = _fold(t.pointwise, bn)
                    w = w[:, :, 0]
                    if r == len(pairs) - 1 and blk.use_res:
                        res = blk.residual
                        wr, br = _fold(res[0].conv, res[1])
                        w, bias = torch.cat([w, wr[:, :, 0]], dim=1), bias + br
                    if w.shape[1] % 8 or cout % 8:
                        raise UnsupportedModel("pointwise widths must be multiples of 8")
                    b["reps"].append(dict(cdw=cdw, wd=_dev16(t.depthwise.weight.detach(), dev), w=_dev16(w, dev),
                                          b=_dev16(bias, dev)))
            else:
                w, bias = _fold(convs[0], pairs[0][1])
                if i == 0:
                    b["w"] = _dev16(w, dev)
                else:
                    if (k * cin) % 8 or cout % 8:
                        raise UnsupportedModel("dense convolution widths must be multiples of 8")
                    b["w"] = _dev16(w.permute(0, 2, 1).reshape(cout, -1), dev)      # [Cout][tap * Cin + cin]
                b["b"] = _dev16(bias, dev)
            self.blocks.append(b)
        head = model.decoder.layers[0]
        self.features = head.in_channels
        if head.out_channels != 5 or head.kernel_size[0] != 1 or self.features % 8:
            raise UnsupportedModel("the decoder must be Conv1d(features -> 5, k1) with features % 8 == 0")
        self.wh = _dev16(head.weight.detach()[:, :, 0], dev)
        self.bh = _dev16(None if head.bias is None else head.bias.detach(), dev)
        self.stride = self.blocks[0]["stride"]
        self._bufs = {}

    # ------------------------------------------------------------------------------------------------
    def frames(self, L):
        return (L - 1) // self.stride + 1

    def _layout(self, i):
        """Input layout of block i >= 1: (buffer role, pitch, column offset of the block input, halo rows per side).  Role
        "io": one of the two ping-pong buffers (block i reads io[i % 2]); role "halo": a zero-haloed buffer of block i's own."""
        b = self.blocks[i]
        if b["residual"]:
            left = b["reps"][-1]["cdw"]
            return "io", left + b["cin"], left, 0
        if not b["separable"] and b["k"] > 1:
            return "halo", b["cin"], 0, b["k"] // 2
        return "io", b["cin"], 0, 0

    def _buffers(self, N, L):
        key = (N, L)
        if key not in self._bufs:
            self._bufs.clear()
            T = self.frames(L)
            M = N * T
            dev, f16 = self.device, torch.float16
            io = [0, 0]
            halo = {}
            for i in range(1, len(self.blocks)):
                role, pitch, _, p = self._layout(i)
                if role == "io":
                    io[i % 2] = max(io[i % 2], M * pitch)
                else:
                    # one per block: its halo rows stay zero (only frame rows are written), and the GEMM reading it writes
                    # elsewhere; the tail covers the k - 1 rows the last chunk's GEMM rows read past the end
                    halo[i] = torch.zeros(N * (T + 2 * p) * pitch + self.blocks[i]["k"] * pitch, dtype=f16, device=dev)
            wide = max([r["cdw"] for b in self.blocks for r in b.get("reps", [])] + [b["cout"] for b in self.blocks])
            bufs = dict(T=T, M=M,
                        io=[torch.empty(n, dtype=f16, device=dev) for n in io],
                        halo=halo,
                        dw=torch.empty(M * wide, dtype=f16, device=dev), h=torch.empty(M * wide, dtype=f16, device=dev),
                        feat=torch.empty(M * self.features, dtype=f16, device=dev),
                        labels=torch.empty(N, T, dtype=torch.uint8, device=dev),
                        probs=torch.empty(N, T, dtype=torch.float32, device=dev))
            self._bufs[key] = bufs
        return self._bufs[key]

    def _dest(self, bufs, i, N, T):
        """Where block i writes its output: (tensor view starting at frame 0 of chunk 0, pitch, rows per chunk)."""
        if i + 1 == len(self.blocks):
            return bufs["feat"], self.features, T
        role, pitch, off, p = self._layout(i + 1)
        buf = bufs["halo"][i + 1] if role == "halo" else bufs["io"][(i + 1) % 2]
        return buf[p * pitch + off:], pitch, T + 2 * p

    def forward(self, x, events=None, **_):
        """x [N, L] (or [N, 1, L]) fp16 -> [N, T, 5] fp16 log-probs."""
        with torch.cuda.device(self.device):
            bufs, N, T = self._encode(x, events)
            out = torch.empty(N, T, 5, dtype=torch.float16, device=self.device)
            with _Stage("head", events):
                native.ctc_head(bufs["feat"], N * T, self.wh, self.bh, bufs["labels"], bufs["probs"], logp=out)
            return out

    def greedy(self, x, events=None):
        """x [N, L] fp16 -> (labels uint8 [N, T], probs fp32 [N, T]) on the device, without the log-probs.  The returned
        tensors are the plan's buffers: the next call with the same shape overwrites them."""
        with torch.cuda.device(self.device):
            bufs, N, T = self._encode(x, events)
            with _Stage("head", events):
                native.ctc_head(bufs["feat"], N * T, self.wh, self.bh, bufs["labels"], bufs["probs"])
            return bufs["labels"], bufs["probs"]

    def _encode(self, x, events):
        if x.dim() == 3:
            x = x[:, 0, :]
        x = x.to(device=self.device, dtype=torch.float16).contiguous()
        N, L = x.shape
        bufs = self._buffers(N, L)
        T, M = bufs["T"], bufs["M"]

        def stage(name):
            return _Stage(name, events)

        def gemm(a, lda, w, bias, dst, ldc, rows, rows_inner, valid, stride_outer, act):
            native.gemm(a, lda, w, bias, dst, ldc, rows, w.shape[0], w.shape[1], act=act, rows_inner=rows_inner,
                        valid_inner=valid, stride_inner=1, stride_outer=stride_outer)

        b0 = self.blocks[0]
        dst, ld, lp = self._dest(bufs, 0, N, T)
        with stage("first_conv"):
            native.conv_first_ex(x, b0["w"], b0["b"], b0["act"], dst, ld, lp, 0, stride=b0["stride"])
        for i in range(1, len(self.blocks)):
            b = self.blocks[i]
            role, pitch, off, p = self._layout(i)
            src = bufs["halo"][i] if role == "halo" else bufs["io"][i % 2]
            dst, ld, lp = self._dest(bufs, i, N, T)
            if not b["separable"]:
                with stage("dense"):      # k > 1: A row n * (T + 2p) + t covers the k frames around frame t
                    rows_inner = T + 2 * p
                    gemm(src, pitch, b["w"], b["b"], dst, ld, N * rows_inner, rows_inner, T, lp, b["act"])
                continue
            cur, cur_ld = src[off:], pitch
            R = len(b["reps"])
            for r, rep in enumerate(b["reps"]):
                last = r == R - 1
                if last and b["residual"]:
                    dw, dw_ld = src, pitch                   # left-hand columns of [depthwise out | block input]
                else:
                    dw, dw_ld = bufs["dw"], rep["cdw"]
                with stage("depthwise"):
                    native.depthwise_conv(cur, cur_ld, rep["wd"], dw, dw_ld, N, T)
                if last:
                    with stage("pointwise"):
                        gemm(dw, dw_ld, rep["w"], rep["b"], dst, ld, M, T, T, lp, b["act"])
                else:
                    with stage("pointwise"):
                        gemm(dw, dw_ld, rep["w"], rep["b"], bufs["h"], b["cout"], M, M, M, 0, b["act"])
                    cur, cur_ld = bufs["h"], b["cout"]
        return bufs, N, T
