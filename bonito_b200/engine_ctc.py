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


def _walk(model):
    """Validate the `Encoder` / `Block` / `TCSConv1d` / `Decoder` tree against the shape rules of the native kernels; one
    dict per block with its (TCSConv1d, BatchNorm1d) pairs, residual modules and shapes, and the head Conv1d."""
    from bonito_b200.ctc.model import Block, TCSConv1d
    blocks = list(model.encoder.encoder)
    if not blocks or not all(isinstance(b, Block) for b in blocks):
        raise UnsupportedModel("native CTC path needs an Encoder of Blocks")
    out = []
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
        cin = pairs[0][0].depthwise.in_channels if separable else convs[0].in_channels
        cout = pairs[-1][1].num_features
        if separable:
            for t, _ in pairs:
                if not depthwise_supported(t.depthwise.in_channels, k):
                    raise UnsupportedModel(f"depthwise convolution C={t.depthwise.in_channels} k{k} has no native kernel")
        out.append(dict(block=blk, pairs=pairs, separable=separable, residual=bool(blk.use_res), act=_ACTS[name], k=k,
                        stride=stride, cin=cin, cout=cout))
    head = model.decoder.layers[0]
    if head.out_channels != 5 or head.kernel_size[0] != 1 or head.in_channels % 8:
        raise UnsupportedModel("the decoder must be Conv1d(features -> 5, k1) with features % 8 == 0")
    return out, head


class CtcPlan:
    supports_slots = False

    def __init__(self, model, device, quantize=False):
        if quantize:
            raise UnsupportedModel("int8 (--quantize) has no native path for the QuartzNet CTC models")
        self.device = dev = torch.device(device)
        walked, head = _walk(model)
        self.blocks = []
        for i, wb in enumerate(walked):
            blk, pairs, k, cin, cout = wb["block"], wb["pairs"], wb["k"], wb["cin"], wb["cout"]
            b = dict(separable=wb["separable"], residual=wb["residual"], act=wb["act"], k=k, stride=wb["stride"], cin=cin,
                     cout=cout, reps=[])
            if wb["separable"]:
                for r, (t, bn) in enumerate(pairs):
                    w, bias = _fold(t.pointwise, bn)
                    w = w[:, :, 0]
                    if r == len(pairs) - 1 and blk.use_res:
                        res = blk.residual
                        wr, br = _fold(res[0].conv, res[1])
                        w, bias = torch.cat([w, wr[:, :, 0]], dim=1), bias + br
                    if w.shape[1] % 8 or cout % 8:
                        raise UnsupportedModel("pointwise widths must be multiples of 8")
                    b["reps"].append(dict(cdw=t.depthwise.in_channels, wd=_dev16(t.depthwise.weight.detach(), dev),
                                          w=_dev16(w, dev), b=_dev16(bias, dev)))
            else:
                w, bias = _fold(pairs[0][0].conv, pairs[0][1])
                if i == 0:
                    b["w"] = _dev16(w, dev)
                else:
                    if (k * cin) % 8 or cout % 8:
                        raise UnsupportedModel("dense convolution widths must be multiples of 8")
                    b["w"] = _dev16(w.permute(0, 2, 1).reshape(cout, -1), dev)      # [Cout][tap * Cin + cin]
                b["b"] = _dev16(bias, dev)
            self.blocks.append(b)
        self.features = head.in_channels
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


# ------------------------------------------------------------------------------------------------------------------------
# Training (train mode, grad enabled): batch-statistics BatchNorm, dropout, and the backward pass
# ------------------------------------------------------------------------------------------------------------------------
class CtcTrainPlan:
    """
    Training forward and backward of the module tree on the GPU, with torch's train-mode semantics under fp16 autocast.

    Forward, per convolution + BatchNorm: the pre-BatchNorm convolution runs on the inference kernels with no bias and no
    activation (`b200_conv_first_fwd_ex`, `b200_depthwise_conv_fwd`, `b200_gemm_fwd_ex`; v2's k15 dense conv over a
    zero-haloed buffer), then `b200_bn_stats` (batch mean and biased variance over the N*T frames, eps and momentum of the
    module, running statistics updated in place) and `b200_bn_act_fwd` (BatchNorm, the residual branch's BatchNorm in a
    residual block, activation, dropout with the block's p).  The residual branch keeps its own statistics, so a residual
    block runs the last pointwise conv and the 1x1 residual conv as two GEMMs.  Operands are fp16 with fp32 accumulation;
    the fp32 master weights are cast to fp16 once per forward.  The head returns fp32 log-probs [N, T, 5].

    Dropout: element (frame, channel) of dropout layer u is kept by a counter-based hash of (seed, u, index); the seed is
    drawn from torch's CPU generator on every forward (Model.forward), so torch.manual_seed makes a run reproducible.
    The keep bits are saved for the backward pass.

    Backward: `b200_ctc_head_bwd`; per BatchNorm `b200_bn_act_bwd` (the activation input recomputed from the saved
    pre-BatchNorm tensors); weight gradients by `b200_wgrad_gemm` (pointwise, residual, dense; the k15 conv in one call
    over the haloed buffer), `b200_depthwise_wgrad` and `b200_conv_first_wgrad`; input gradients by the forward kernels:
    `b200_gemm_fwd_ex` with the weight transposed (the k15 conv over a haloed dz with the taps reversed) and
    `b200_depthwise_conv_fwd` with the taps reversed.  The two gradients into a residual block's input are summed inside
    the next `b200_bn_act_bwd` (depthwise path first).  Every kernel is deterministic, so two identical steps give
    bitwise-equal gradients.

    Everything saved lives in the object `forward` returns (held by the autograd graph), never in plan buffers, so any
    number of forwards may precede their backwards.
    """

    def __init__(self, model):
        self.walked, self.head = _walk(model)
        self.params = []
        for wb in self.walked:
            blk = wb["block"]
            drops = [m.p for m in list(blk.conv) + list(blk.activation) if isinstance(m, torch.nn.Dropout)]
            if len(set(drops)) > 1:
                raise UnsupportedModel("the dropouts of a block must share p")
            wb["p"] = drops[0] if drops else 0.0
            for t, bn in wb["pairs"]:
                self._check_bn(bn)
            if wb["residual"]:
                self._check_bn(blk.residual[1])
            if wb["separable"] and wb["cout"] % 8:
                raise UnsupportedModel("pointwise widths must be multiples of 8")
        for p in model.parameters():
            if p.dtype != torch.float32:
                raise UnsupportedModel("training needs fp32 master weights (the model was converted to another dtype)")
            self.params.append(p)
        self._index = {id(p): i for i, p in enumerate(self.params)}
        self.stride = self.walked[0]["stride"]
        self.features = self.head.in_channels

    @staticmethod
    def _check_bn(bn):
        if not (bn.affine and bn.track_running_stats and bn.momentum is not None):
            raise UnsupportedModel("training needs affine BatchNorm1d with running statistics and a momentum")

    # ------------------------------------------------------------------------------------------------
    def forward(self, x, seed):
        """x [N, L] (or [N, 1, L]) -> (log-probs fp32 [N, T, 5], saved state for `backward`)."""
        if x.dim() == 3:
            x = x[:, 0, :]
        dev = x.device
        x = x.to(torch.float16).contiguous()
        N, L = x.shape
        T = (L - 1) // self.stride + 1
        M = N * T
        f16 = torch.float16
        S = dict(x=x, N=N, T=T, M=M, seed=int(seed), blocks=[], unit=0)

        def empty(rows, c):
            return torch.empty(rows, c, dtype=f16, device=dev)

        def bn_unit(z, bn, act, p, dst, ldo, lpo, res=None):
            """stats of z (and of the residual branch's zr), then BatchNorm -> act -> dropout into dst."""
            C = bn.num_features
            rec = dict(z=z, bn=bn, act=act, p=p, unit=S["unit"], res=res)
            S["unit"] += 1
            for key, (zz, b) in (("", (z, bn)),) + ((("_r", res),) if res is not None else ()):
                mean = torch.empty(C, dtype=torch.float32, device=dev)
                invstd = torch.empty_like(mean)
                native.bn_stats(zz, C, M, C, b.eps, b.momentum, mean, invstd, b.running_mean, b.running_var)
                b.num_batches_tracked.add_(1)
                rec["mean" + key], rec["invstd" + key] = mean, invstd
            rec["mask"] = torch.empty(M, C // 8, dtype=torch.uint8, device=dev) if p > 0 else None
            native.bn_act_fwd(self._bn_args(rec, S), dst, ldo, lpo)
            return rec

        def out_buffer(i, C):
            """(tensor, view at frame 0 of chunk 0, pitch, rows per chunk) of block i's output: a zero-haloed buffer when
            block i + 1 is a dense k > 1 conv, compact rows otherwise."""
            if i + 1 < len(self.walked):
                nb = self.walked[i + 1]
                if not nb["separable"] and nb["k"] > 1:
                    p = nb["k"] // 2
                    buf = torch.zeros(N * (T + 2 * p) * C + nb["k"] * C, dtype=f16, device=dev)
                    return buf, buf[p * C:], C, T + 2 * p
            buf = empty(M, C)
            return buf, buf, C, T

        h = None      # (tensor, pitch) of the current block input
        for i, wb in enumerate(self.walked):
            blk, act, p = wb["block"], wb["act"], wb["p"]
            cout = wb["cout"]
            out, out_v, ld, lp = out_buffer(i, cout)
            rec = dict(kind=None, out=(out, out_v, ld, lp))
            if i == 0:
                conv, bn = wb["pairs"][0]
                w16 = conv.conv.weight.detach().to(f16).contiguous()
                z = empty(M, cout)
                native.conv_first_ex(x, w16, None, native.ACT_NONE, z, cout, T, 0, stride=self.stride)
                rec.update(kind="first", w=conv.conv.weight, k=wb["k"], bn=bn_unit(z, bn, act, p, out_v, ld, lp))
            elif not wb["separable"]:
                conv, bn = wb["pairs"][0]
                k, cin = wb["k"], wb["cin"]
                w = conv.conv.weight.detach()
                w16 = w.permute(0, 2, 1).reshape(cout, k * cin).to(f16).contiguous()      # [Cout][tap * Cin + cin]
                z = empty(M, cout)
                pd = k // 2
                rows_inner = T + 2 * pd
                native.gemm(h[0], cin, w16, None, z, cout, N * rows_inner, cout, k * cin, rows_inner=rows_inner, valid_inner=T,
                            stride_outer=T)
                rec.update(kind="dense", conv=conv.conv, w16=w16, k=k, cin=cin, x=h[0], bn=bn_unit(z, bn, act, p, out_v, ld, lp))
            else:
                reps = []
                hin, R = h[0], len(wb["pairs"])
                for r, (tcs, bn) in enumerate(wb["pairs"]):
                    cdw = tcs.depthwise.in_channels
                    wd16 = tcs.depthwise.weight.detach().to(f16).contiguous()
                    wp16 = tcs.pointwise.weight.detach()[:, :, 0].to(f16).contiguous()
                    d = empty(M, cdw)
                    native.depthwise_conv(hin, cdw, wd16, d, cdw, N, T)
                    z = empty(M, cout)
                    native.gemm(d, cdw, wp16, None, z, cout, M, cout, cdw)
                    rep = dict(tcs=tcs, h=hin, d=d, wd16=wd16, wp16=wp16, cdw=cdw)
                    if r == R - 1:
                        res = None
                        if wb["residual"]:
                            rconv, rbn = blk.residual[0].conv, blk.residual[1]
                            wr16 = rconv.weight.detach()[:, :, 0].to(f16).contiguous()
                            zr = empty(M, cout)
                            native.gemm(h[0], wb["cin"], wr16, None, zr, cout, M, cout, wb["cin"])
                            res = (zr, rbn)
                            rec.update(rconv=rconv, wr16=wr16, x=h[0])
                        rep["bn"] = bn_unit(z, bn, act, p, out_v, ld, lp, res=res)
                    else:
                        hnext = empty(M, cout)
                        rep["bn"] = bn_unit(z, bn, act, p, hnext, cout, T)
                        hin = hnext
                    reps.append(rep)
                rec.update(kind="separable", reps=reps, cin=wb["cin"])
            S["blocks"].append(rec)
            h = (out, ld)
        feat = h[0]
        wh16 = self.head.weight.detach()[:, :, 0].to(f16).contiguous()
        bh16 = None if self.head.bias is None else self.head.bias.detach().to(f16).contiguous()
        logp = torch.empty(M, 5, dtype=torch.float32, device=dev)
        native.ctc_head_train_fwd(feat, M, wh16, bh16, logp)
        S.update(feat=feat, wh16=wh16, logp=logp)
        return logp.view(N, T, 5), S

    @staticmethod
    def _bn_args(rec, S):
        bn = rec["bn"]
        res = None
        if rec["res"] is not None:
            zr, rbn = rec["res"]
            res = (zr, zr.shape[1], rec["mean_r"], rec["invstd_r"], rbn.weight.detach(), rbn.bias.detach())
        return native.bn_act_struct(S["M"], bn.num_features, S["T"], rec["act"], rec["p"], S["seed"], rec["unit"], rec["z"],
                                    rec["z"].shape[1], rec["mean"], rec["invstd"], bn.weight.detach(), bn.bias.detach(),
                                    residual=res, mask=rec["mask"])

    # ------------------------------------------------------------------------------------------------
    def backward(self, S, g):
        """g = dL/dlogp [N, T, 5] -> gradients of `self.params` (fp32, None for parameters the model does not use)."""
        N, T, M = S["N"], S["T"], S["M"]
        dev = g.device
        f16 = torch.float16
        grads = [None] * len(self.params)

        def put(param, value):
            grads[self._index[id(param)]] = value.view(param.shape)

        def zeros32(*shape):
            return torch.empty(*shape, dtype=torch.float32, device=dev)

        g = g.to(torch.float32).contiguous()
        F = self.features
        dfeat = torch.empty(M, F, dtype=f16, device=dev)
        dwh, dbh = zeros32(5, F), zeros32(5)
        native.ctc_head_bwd(S["feat"], M, S["wh16"], S["logp"], g.view(M, 5), dwh, dbh, dfeat)
        put(self.head.weight, dwh)
        if self.head.bias is not None:
            put(self.head.bias, dbh)

        dy = (dfeat, F, None, 0)      # gradient at the current block's output: (dy, ldy, dy2, ldy2), compact rows

        def bn_bwd(rec, dy, dz_halo=None):
            """dz (and dzr) of one BatchNorm unit; BatchNorm parameter gradients stored."""
            bn, C = rec["bn"], rec["bn"].num_features
            dgamma, dbeta = zeros32(C), zeros32(C)
            if dz_halo is None:
                dz = torch.empty(M, C, dtype=f16, device=dev)
                dz_v, ldo, lpo = dz, C, T
            else:
                dz, dz_v, ldo, lpo = dz_halo
            kw = {}
            dzr = None
            if rec["res"] is not None:
                rbn = rec["res"][1]
                dzr = torch.empty(M, C, dtype=f16, device=dev)
                kw = dict(dgamma_r=zeros32(C), dbeta_r=zeros32(C), dzr=dzr)
            native.bn_act_bwd(self._bn_args(rec, S), dy[0], dy[1], dgamma, dbeta, dz_v, ldo, lpo, dy2=dy[2], ldy2=dy[3], **kw)
            put(bn.weight, dgamma)
            put(bn.bias, dbeta)
            if dzr is not None:
                put(rbn.weight, kw["dgamma_r"])
                put(rbn.bias, kw["dbeta_r"])
            return dz, dzr

        for i in range(len(self.walked) - 1, -1, -1):
            rec = S["blocks"][i]
            wb = self.walked[i]
            cout = wb["cout"]
            if rec["kind"] == "first":
                dz, _ = bn_bwd(rec["bn"], dy)
                dw = zeros32(*rec["w"].shape)
                native.conv_first_wgrad(dz, cout, S["x"], self.stride, dw)
                put(rec["w"], dw)
            elif rec["kind"] == "dense":
                k, cin = rec["k"], rec["cin"]
                pd = k // 2
                rows_inner = T + 2 * pd
                if k > 1:
                    buf = torch.zeros(N * rows_inner * cout + k * cout, dtype=f16, device=dev)
                    dz_halo = (buf, buf[pd * cout:], cout, rows_inner)
                    dz, _ = bn_bwd(rec["bn"], dy, dz_halo)
                    dz_v = dz_halo[1]
                else:
                    dz, _ = bn_bwd(rec["bn"], dy)
                    dz_v = dz
                dw = zeros32(cout, k * cin)
                native.wgrad_gemm(dz_v, cout, rec["x"], cin, N * rows_inner, cout, k * cin, dw, rows_inner=rows_inner,
                                  valid_inner=T, lpz=rows_inner)
                put(rec["conv"].weight, dw.view(cout, k, cin).permute(0, 2, 1).contiguous())
                # dX[t] = sum_j dz[t - pd + j] W[:, :, k - 1 - j]: the haloed dz against the taps in reverse order
                wt = rec["conv"].weight.detach().flip(-1).permute(1, 2, 0).reshape(cin, k * cout).to(f16).contiguous()
                dx = torch.empty(M, cin, dtype=f16, device=dev)
                native.gemm(dz, cout, wt, None, dx, cin, N * rows_inner, cin, k * cout, rows_inner=rows_inner, valid_inner=T,
                            stride_outer=T)
                dy = (dx, cin, None, 0)
            else:
                reps = rec["reps"]
                dh = None
                dzr = None
                for r in range(len(reps) - 1, -1, -1):
                    rep = reps[r]
                    dz, dzr_r = bn_bwd(rep["bn"], dy if r == len(reps) - 1 else (dh, cout, None, 0))
                    if dzr_r is not None:
                        dzr = dzr_r
                    cdw = rep["cdw"]
                    dw = zeros32(cout, cdw)
                    native.wgrad_gemm(dz, cout, rep["d"], cdw, M, cout, cdw, dw)
                    put(rep["tcs"].pointwise.weight, dw)
                    dd = torch.empty(M, cdw, dtype=f16, device=dev)
                    native.gemm(dz, cout, rep["wp16"].t().contiguous(), None, dd, cdw, M, cdw, cout)
                    dwd = zeros32(*rep["tcs"].depthwise.weight.shape)
                    native.depthwise_wgrad(dd, cdw, rep["h"], cdw, N, T, dwd)
                    put(rep["tcs"].depthwise.weight, dwd)
                    dh = torch.empty(M, cdw, dtype=f16, device=dev)
                    native.depthwise_conv(dd, cdw, rep["wd16"].flip(-1).contiguous(), dh, cdw, N, T)
                cin = rec["cin"]
                if dzr is not None:
                    dw = zeros32(cout, cin)
                    native.wgrad_gemm(dzr, cout, rec["x"], cin, M, cout, cin, dw)
                    put(rec["rconv"].weight, dw)
                    dxr = torch.empty(M, cin, dtype=f16, device=dev)
                    native.gemm(dzr, cout, rec["wr16"].t().contiguous(), None, dxr, cin, M, cin, cout)
                    dy = (dh, cin, dxr, cin)
                else:
                    dy = (dh, cin, None, 0)
        return grads


class CtcTrainFunction(torch.autograd.Function):
    """Autograd node of `CtcTrainPlan`: forward(plan, seed, x, *plan.params) -> fp32 log-probs [N, T, 5]."""

    @staticmethod
    def forward(ctx, plan, seed, x, *params):
        logp, saved = plan.forward(x, seed)
        ctx.plan, ctx.saved = plan, saved
        return logp

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        grads = ctx.plan.backward(ctx.saved, g)
        ctx.saved = None
        return (None, None, None, *grads)
