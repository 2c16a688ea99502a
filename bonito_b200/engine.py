"""
Plan builder + executor for the LSTM-CRF encoder (the `bonito.crf` fast / hac / LSTM sup models; LSTM widths 96, 128, 256,
384, 768, 1024).

`compile_lstm_crf(encoder)` walks a `bonito_b200.nn` module tree of the shape the reference's
configs describe (`bonito/models/configs/dna_r10.4.1@v4.3.toml`,
`bonito/crf/model.py:150-162`):

    Convolution(1->C1,k5) [, Clamp] , Convolution(C1->C2,k5) [, Clamp] , Convolution(C2->H,kW,stride s) [, Clamp]
    Permute([2,0,1]) , LSTM x L (alternating reverse) [, Linear(H->B)] , LinearCRFEncoder [, Clamp]

(LinearCRFEncoder: a plain linear head followed by a Clamp layer, as in the v4+ configs, or the old-style head with
activation = "tanh" and / or a scale and no Clamp) and packs the weights into the operand layouts of the sm_90a kernels
(include/bonito_b200.h).  This is the native swap-in the reference performs in `Model.use_koi`
(`bonito/crf/model.py:240-246`, koi.lstm.update_graph); like koi it returns scores as `[N, T, C]` fp16 without the blank
column when the head has a fixed blank_score.  A head without one (dna_r9.4.1@v3) learns its blank scores: the scores
are then `[N, T, 5 * 4^k]` in the CTC_CRF order [state][stay, m0..m3] (b200_crf_decode_lb).  A Clamp behind a (swish)
convolution (dna_r10.4.1@v4.0) is fused into its epilogue (B200_ACT_SWISH_CLAMP), the Linear in front of the head is one
more GEMM; these layers and learned blank scores run on the wide layout (H = 768, 1024) only.  Anything else raises
`UnsupportedModel`.

Every layout shares the front end: the fused conv1 + conv2 stem writes `[N][Lp][C2]` channels last, and the strided conv3 is
one GEMM over the overlapping-row view of it.  The LSTM width picks one of three activation layouts (`LstmCrfPlan.forward`):

* Tile layout, width 384 (hac, the headline path; `forward_tiles`): activations tile-major `[tile][T][64][H]`; the fused
  wgmma LSTM kernel (lstm_fused_tile.cu: one 8-CTA cluster per 64-chunk tile, 8 clusters for 512 chunks), which computes
  the input projection inside the recurrence, runs the LSTM stack in chains of consecutive tiles, each chain on a stream
  of its own through all the layers (b200_lstm_crf_lstm_fwd).  Under
  `--quantize` the input projection is an int8 GEMM into gate pre-activations `[tile][T][8][64][192]` instead, followed by
  the unfused recurrent kernel (lstm_rec_tile.cu).  The whole encoder is one C call (`b200_lstm_crf_fwd`) unless per-kernel
  events, intermediate activations, another GEMM implementation or the int8 input projection ask for the launches one at
  a time.  Buffers are cached per (batch, chunk
  length, slot): `slot` selects one of several independent buffer sets, so that consecutive batches can be in flight on
  different streams (`score_batches`, bench.py).

* Generic layout, widths 96, 128 and 256, and 384 under `B200_LSTM_TILE=0` (`forward_generic`): the `mma.sync` recurrent
  kernel on activations `[T][n][H]` and gate pre-activations `[T][n][4H]` of a tile of n chunks.  A batch of more than
  one 32-chunk tile runs its tiles on streams of their own, so that the GEMMs of one tile fill the SMs the recurrences of
  the others leave free; a single tile runs on the current stream.

* Wide layout, widths 768 and 1024 (`forward_wide`: dna_r9.4.1@v3.1, dna_r10.4.1@v4.3): W_hh does not fit the shared memory
  of one cluster, so the recurrence runs on the grid-wide kernel (lstm_rec_wide.cu: H / 8 co-resident CTAs, one cooperative
  launch per layer); activations `[T][N][H]`, gate pre-activations `[T][H/8][N][32]`, layer by layer on the current
  stream, one buffer set (no slots), no int8 input projection; the output of the Linear in front of the head, if any, is
  `[T][N][B]`.
"""

import os
import threading

import torch

from bonito_b200 import native
from bonito_b200 import nn as bnn

_ACT_CODES = {None: native.ACT_NONE, "swish": native.ACT_SWISH, "tanh": native.ACT_TANH}
WIDTHS = (96, 128, 256, 384, 768, 1024)     # LSTM hidden sizes with a native recurrent kernel


class UnsupportedModel(NotImplementedError):
    pass


def _act_code(module):
    if module is None:
        return native.ACT_NONE
    name = getattr(module, "name", None)
    if name not in _ACT_CODES:
        raise UnsupportedModel(f"activation {module!r} has no native kernel")
    return _ACT_CODES[name]


def _folded_conv(layer):
    """(weight, bias) of a Convolution with any BatchNorm folded in (bonito/nn.py:447-454)."""
    conv = layer.conv
    if layer.norm is not None:
        if not isinstance(layer.norm, bnn.BatchNorm):
            raise UnsupportedModel(f"norm {layer.norm!r} has no native kernel")
        conv = torch.nn.utils.fusion.fuse_conv_bn_eval(conv.eval(), layer.norm.bn.eval())
    return conv.weight.detach(), None if conv.bias is None else conv.bias.detach()


def _conv_act(conv, clamp):
    """(activation code, lo, hi) of a Convolution and the Clamp layer behind it (None: no Clamp)."""
    act = _act_code(conv.activation)
    if clamp is None:
        return act, 0.0, 0.0
    if act != native.ACT_SWISH:
        raise UnsupportedModel(f"a Clamp after a convolution is supported behind a swish activation; got {conv.activation!r}")
    return native.ACT_SWISH_CLAMP, float(clamp.min), float(clamp.max)


def _parse_stack(layers):
    """
    Split an encoder into (convs, clamps behind them, lstms, bottleneck Linear or None, LinearCRFEncoder, head clamps) if it is
        [Convolution, Clamp?] x 3, Permute([2, 0, 1]), LSTM x L (L >= 1), Linear?, LinearCRFEncoder, Clamp?
    and raise UnsupportedModel otherwise.
    """
    names = [type(m).__name__ for m in layers]
    err = UnsupportedModel("native LSTM-CRF path needs [Convolution, Clamp?] x 3, Permute([2, 0, 1]), LSTM x L, Linear?, "
                           f"LinearCRFEncoder, Clamp?; got {names}")
    i = 0

    def take(cls):
        nonlocal i
        if i < len(layers) and isinstance(layers[i], cls):
            i += 1
            return layers[i - 1]
        return None

    convs, conv_clamps = [], []
    for _ in range(3):
        convs.append(take(bnn.Convolution))
        conv_clamps.append(take(bnn.Clamp))
    permute = take(bnn.Permute)
    if None in convs or permute is None or list(permute.dims) != [2, 0, 1]:
        raise err
    lstms = []
    while (m := take(bnn.LSTM)) is not None:
        lstms.append(m)
    bottleneck = take(bnn.Linear)
    crf = take(bnn.LinearCRFEncoder)
    head_clamp = take(bnn.Clamp)
    if not lstms or crf is None or i != len(layers):
        raise err
    return convs, conv_clamps, lstms, bottleneck, crf, [] if head_clamp is None else [head_clamp]


def _dev16(t, device):
    return None if t is None else t.to(device=device, dtype=torch.float16).contiguous()


class _Stage:
    """Context manager recording a CUDA event pair around one kernel launch on `stream` (default: the current stream); no-op
    without a sink."""

    def __init__(self, name, sink, stream=None):
        self.name, self.sink, self.stream = name, sink, stream

    def __enter__(self):
        if self.sink is not None:
            self.start = torch.cuda.Event(enable_timing=True)
            self.start.record(self.stream)

    def __exit__(self, *exc):
        if self.sink is not None:
            end = torch.cuda.Event(enable_timing=True)
            end.record(self.stream)
            self.sink.append((self.name, self.start, end))
        return False


class LstmCrfPlan:
    """Packed weights + cached buffers for one LSTM-CRF encoder on one device."""

    def __init__(self, encoder, device, quantize=False):
        convs, conv_clamps, lstms, bottleneck, crf, clamps = _parse_stack(list(encoder.children()))
        self.device = torch.device(device)

        # --- conv stem (conv1 + conv2) -------------------------------------------------------
        c1, c2, c3 = convs
        for c in (c1, c2):
            k = c.conv.kernel_size[0]
            if c.conv.stride[0] != 1 or c.conv.padding[0] != k // 2 or k % 2 == 0:
                raise UnsupportedModel("conv stem layers must be stride 1 with 'same' padding")
        if c1.conv.in_channels != 1:
            raise UnsupportedModel("the encoder must take a single input feature")
        (self.act1, lo1, hi1), (self.act2, lo2, hi2), (self.act3, self.lo3, self.hi3) = (
            _conv_act(c, clamp) for c, clamp in zip(convs, conv_clamps))
        # bounds of the stem activations (B200_ACT_SWISH_CLAMP), None: no clamp in the stem
        self.stem_bounds = (lo1, hi1, lo2, hi2) if any(conv_clamps[:2]) else None
        w1, b1 = _folded_conv(c1)
        w2, b2 = _folded_conv(c2)
        self.w1, self.b1 = _dev16(w1, device), _dev16(b1, device)
        self.w2, self.b2 = _dev16(w2, device), _dev16(b2, device)

        # --- strided conv as GEMM: weight [H][C2][K3] -> [H][K3*C2], k = tap*C2 + cin -------
        w3, b3 = _folded_conv(c3)
        self.hidden, self.c2, self.k3 = w3.shape
        self.s3, self.pad3 = c3.conv.stride[0], c3.conv.padding[0]
        self.w3 = _dev16(w3.permute(0, 2, 1).reshape(self.hidden, -1), device)
        self.b3 = _dev16(b3, device)
        if (self.k3 * self.c2) % 8 or (self.s3 * self.c2) % 8:
            raise UnsupportedModel("strided conv window/stride must be multiples of 8 elements")

        # --- LSTM stack ------------------------------------------------------------------------
        H = self.hidden
        self.wide = 0                                      # > 0: CTAs of the wide recurrent kernel (H = 768, 1024)
        if native.lstm_cluster_size(H) == 0:
            self.wide = native.lstm_wide_ctas(H)
            if self.wide == 0:
                raise UnsupportedModel(f"LSTM hidden size {H} has no native kernel (supported: {', '.join(map(str, WIDTHS))})")
            resident = native.lstm_wide_resident(H, self.device)
            if resident < self.wide:
                raise UnsupportedModel(f"the wide LSTM kernel for hidden size {H} needs {self.wide} co-resident CTAs (one per "
                                       f"SM); this device holds {resident}")
        # H = 384: tile-layout recurrent kernel (64-chunk tiles, 8-CTA clusters, wgmma)
        self.tile = native.lstm_tile_chunks(H)            # 0: only the generic-layout kernel exists for this width
        self.tile_cs = native.lstm_tile_cluster(H)
        unit = torch.arange(H)
        perm_ih = (torch.arange(4)[None, :] * H + unit[:, None]).reshape(-1)          # [unit][gate]
        perm_hh = (torch.arange(H // 8)[:, None, None] * 8 + torch.arange(4)[None, :, None] * H
                   + torch.arange(8)[None, None, :]).reshape(-1)                      # [unit/8][gate][unit%8]
        self.lstm = []
        for m in lstms:
            r = m.rnn
            if r.hidden_size != H or r.input_size != H or r.num_layers != 1 or r.bidirectional:
                raise UnsupportedModel("native LSTM path needs single-layer unidirectional LSTMs of equal width")
            bias = torch.zeros(4 * H, dtype=torch.float32)
            if r.bias:
                bias = r.bias_ih_l0.detach().float().cpu() + r.bias_hh_l0.detach().float().cpu()
            self.lstm.append(dict(
                wih=_dev16(r.weight_ih_l0.detach().cpu()[perm_ih], device),
                bias=_dev16(bias[perm_ih], device),
                whh=_dev16(r.weight_hh_l0.detach().cpu()[perm_hh], device),
                reverse=bool(m.reverse),
            ))
            if quantize:
                # --quantize (reference: koi's int8 LSTM, bonito/crf/model.py:245): the input projection runs on int8 tensor
                # cores.  Weights: symmetric per-row int8; activations: LSTM inputs live in (-1, 1) (tanh / o*tanh(c)), fixed
                # scale 127.  gx = (q_x . q_w) * s_w / 127 + bias.  The recurrent weights and the h exchange stay fp16.
                w = r.weight_ih_l0.detach().float().cpu()[perm_ih]
                s_w = w.abs().amax(dim=1).clamp(min=1e-8) / 127.0
                self.lstm[-1]["wih_q"] = torch.round(w / s_w[:, None]).clamp(-127, 127).to(torch.int8).to(device).contiguous()
                self.lstm[-1]["wih_scale"] = (s_w / 127.0).to(device=device, dtype=torch.float32).contiguous()
        self.quantize = bool(quantize)
        if self.tile and len(self.lstm) > native.MAX_LSTM_LAYERS:
            raise UnsupportedModel(f"the tile-layout LSTM path runs at most {native.MAX_LSTM_LAYERS} layers; got {len(self.lstm)}")
        if self.quantize and not (self.tile and H % 16 == 0):
            raise UnsupportedModel("the int8 input projection (--quantize) needs the tile-layout LSTM path (hidden size 384)")

        # --- bottleneck Linear(H -> B) in front of the head (dna_r10.4.1@v4.0) ----------------------
        self.wb = self.bb = None
        self.head_in = H                                    # input width of the CRF head GEMM
        if bottleneck is not None:
            lin = bottleneck.linear
            if lin.in_features != H or lin.out_features % 8:
                raise UnsupportedModel(f"the Linear in front of the CRF head must map the LSTM width {H} to a multiple of 8 "
                                       f"features; got {lin.in_features} -> {lin.out_features}")
            self.wb = _dev16(lin.weight.detach(), device)
            self.bb = _dev16(None if lin.bias is None else lin.bias.detach(), device)
            self.head_in = lin.out_features

        # --- linear CRF head (+ clamp) ---------------------------------------------------------
        if crf.permute is not None:
            raise UnsupportedModel("native LinearCRFEncoder supports permute=None")
        crf_act = _act_code(crf.activation)
        if crf_act not in (native.ACT_NONE, native.ACT_TANH) or ((crf_act != native.ACT_NONE or crf.scale is not None) and clamps):
            raise UnsupportedModel("native LinearCRFEncoder supports tanh and / or a scale (old-style configs), or a Clamp layer "
                                   "behind a plain linear head (v4+ configs)")
        self.n_base, self.state_len = crf.n_base, crf.state_len
        # blank_score None: learned blank scores, the head emits [state][stay, m0..m3] (5 * 4^k columns, b200_crf_decode_lb)
        self.blank_score = None if crf.blank_score is None else float(crf.blank_score)
        self.wl = _dev16(crf.linear.weight.detach(), device)
        self.bl = _dev16(None if crf.linear.bias is None else crf.linear.bias.detach(), device)
        self.n_scores = self.wl.shape[0]
        if self.wl.shape[1] != self.head_in:
            raise UnsupportedModel(f"the CRF head takes {self.wl.shape[1]} features; the layer before it gives {self.head_in}")
        new_layers = [name for name, used in (("a Clamp after a convolution", any(conv_clamps)),
                                              ("a Linear in front of the CRF head", bottleneck is not None),
                                              ("learned blank scores", self.blank_score is None)) if used]
        if new_layers and not self.wide:
            raise UnsupportedModel(f"{' and '.join(new_layers)} run on the wide LSTM path only (hidden size 768 or 1024); "
                                   f"this model has hidden size {H}")
        if clamps:
            self.act_l, self.lo, self.hi = native.ACT_CLAMP, float(clamps[0].min), float(clamps[0].max)
        elif crf_act == native.ACT_TANH and crf.scale is not None:     # e.g. the dna_r9.4.1 configs: tanh, scale 5.0
            self.act_l, self.lo, self.hi = native.ACT_TANH_SCALE, float(crf.scale), 0.0
        elif crf.scale is not None:
            self.act_l, self.lo, self.hi = native.ACT_SCALE, float(crf.scale), 0.0
        else:
            self.act_l, self.lo, self.hi = crf_act, 0.0, 0.0
        self._bufs = {}
        self._chain_streams = {}    # slot -> streams of the LSTM stack's tile chains 1.. (b200_lstm_crf_lstm_fwd)
        self._wide_pending = None   # (event, pinned status words) of the last wide-path forward, checked by the next call

    # ------------------------------------------------------------------------------------------
    def frames(self, L):
        return (L + 2 * self.pad3 - self.k3) // self.s3 + 1

    @property
    def supports_slots(self):
        """Independent buffer sets (several batches in flight) exist for the tile layout only."""
        return bool(self.tile) and os.environ.get("B200_LSTM_TILE", "1") != "0"

    TILE = 32  # chunks per tile of the generic layout (one recurrent cluster each)

    def _buffers(self, layout, N, L, slot=0):
        """
        Work buffers of `layout` ("generic", "tile" or "wide") for N chunks of L samples.  Buffer sets of another layout or
        geometry are dropped; the slots of one layout and geometry stay side by side (batches in flight).
        """
        key = (layout, N, L, slot)
        if key in self._bufs:
            return self._bufs[key]
        for k in [k for k in self._bufs if k[:3] != key[:3]]:
            del self._bufs[k]
        T = self.frames(L)
        need = max(self.pad3 + L, (T - 1) * self.s3 + self.k3)
        Tp = -(-need // self.s3)
        Lp = Tp * self.s3
        dev, f16, H = self.device, torch.float16, self.hidden
        tail = self.k3 * self.c2  # the last window of the overlapping-row view reads past row N*Tp-1
        b = dict(T=T, Tp=Tp, Lp=Lp, stem=torch.empty(N * Lp * self.c2 + tail, dtype=f16, device=dev))
        b["stem"][-tail:].zero_()
        if layout == "generic":
            # flat: the tile of chunks [n0, n0 + nb) is [T][nb][.] at element n0*T*H of ya / yb (n0*T*4H of gx)
            nt = -(-N // self.TILE)
            b.update(ya=torch.empty(N * T * H, dtype=f16, device=dev), yb=torch.empty(N * T * H, dtype=f16, device=dev),
                     gx=torch.empty(N * T * 4 * H, dtype=f16, device=dev),
                     streams=_LazyStreams(dev, nt), start=torch.cuda.Event(), done=[torch.cuda.Event() for _ in range(nt)])
        elif layout == "tile":
            TB, CS = self.tile, self.tile_cs
            nt = -(-N // TB)
            b.update(
                nt=nt,
                # zero-filled once: rows of chunks beyond the batch (last tile) are never written and must stay finite
                ya=torch.zeros(nt, T, TB, H, dtype=f16, device=dev),
                yb=torch.zeros(nt, T, TB, H, dtype=f16, device=dev),
                # gate pre-activations of the int8 input projection; the fp16 layers compute them inside the recurrence
                gx=torch.zeros(nt, T, CS, TB, 4 * H // CS, dtype=f16, device=dev) if self.quantize else None,
                yq=torch.empty(nt * T * TB * H, dtype=torch.int8, device=dev) if self.quantize else None,
                # staging of the recurrent kernel's h all-gather: one region per tile (the clusters run concurrently)
                hx=torch.empty(nt, native.lstm_rec_tile_workspace_bytes(TB), dtype=torch.uint8, device=dev),
                # kept per slot for the life of the plan: a buffer set of another geometry reuses them
                chains=self._chain_streams.setdefault(
                    slot, [native.new_stream(dev) for _ in range(native.LSTM_CHAINS - 1)]),
            )
        else:
            ws = torch.empty(native.lstm_rec_wide_workspace_bytes(N, H), dtype=torch.uint8, device=dev)
            off = native.lstm_rec_wide_status_offset(N, H)
            b.update(
                ya=torch.empty(T, N, H, dtype=f16, device=dev),
                yb=torch.empty(T, N, H, dtype=f16, device=dev),
                gx=torch.empty(T, self.wide, N, 4 * H // self.wide, dtype=f16, device=dev),
                yl=None if self.wb is None else torch.empty(T, N, self.head_in, dtype=f16, device=dev),
                ws=ws, ws_status=ws[off:off + 4].view(torch.int32),
                status=torch.zeros(len(self.lstm), dtype=torch.int32, device=dev),
            )
        self._bufs[key] = b
        return b

    # ------------------------------------------------------------------------------------------
    # front end, shared by the three layouts
    # ------------------------------------------------------------------------------------------
    def _input(self, x):
        """[N, 1, L] or [N, L] -> contiguous fp16 [N, L] on the plan's device."""
        if x.dim() == 3:
            x = x[:, 0, :]
        return x.to(device=self.device, dtype=torch.float16).contiguous()

    def _stem(self, x, b, events, feats):
        """conv1 + conv2 into b["stem"] ([N][Lp][C2], channels last); `feats` (a dict or None) gets the "stem" activations."""
        N, L = x.shape
        Lp = b["Lp"]
        with _Stage("conv_stem", events):
            native.conv_stem(x, self.w1, self.b1, self.act1, self.w2, self.b2, self.act2, b["stem"], Lp, self.pad3,
                             bounds=self.stem_bounds)
        if feats is not None:
            feats["stem"] = b["stem"][:N * Lp * self.c2].view(N, Lp, self.c2)[:, self.pad3:self.pad3 + L].clone()

    def _conv_gemm(self, b, n0, nb, dst, events, gemm_impl, stream=None, **rows):
        """The strided conv of chunks [n0, n0 + nb) as one GEMM: rows r = n*Tp + t are windows of k3*c2 stem elements, s3*c2
        apart; `rows` maps them into `dst` (b200_gemm_fwd_ex)."""
        with _Stage("conv_gemm", events, stream):
            native.gemm(b["stem"][n0 * b["Lp"] * self.c2:], self.s3 * self.c2, self.w3, self.b3, dst, self.hidden,
                        nb * b["Tp"], self.hidden, self.k3 * self.c2, act=self.act3, lo=self.lo3, hi=self.hi3,
                        rows_inner=b["Tp"], valid_inner=b["T"], stride_outer=1, impl=gemm_impl, stream=stream, **rows)

    # ------------------------------------------------------------------------------------------
    # generic layout: tiles of n chunks, activations [T][n][H], gate pre-activations [T][n][4H]
    # ------------------------------------------------------------------------------------------
    def forward_generic(self, x, out=None, gemm_impl=native.GEMM_AUTO, events=None, return_features=False, tiled=None):
        """
        Forward in the generic layout.  `tiled` (default: when the batch has more than one tile): 32-chunk tiles, each on a
        stream of its own and all started behind the stem; otherwise the batch is one tile on the current stream.
        Intermediate activations (`return_features`) are taken from the single-tile schedule.
        """
        x = self._input(x)
        N, L = x.shape
        H, TB = self.hidden, self.TILE
        b = self._buffers("generic", N, L)
        T = b["T"]
        if out is None:
            out = torch.empty(N, T, self.n_scores, dtype=torch.float16, device=self.device)
        feats = {} if return_features else None
        tiled = (N > TB if tiled is None else tiled) and not return_features
        tiles = [(n0, min(TB, N - n0), b["streams"][n0 // TB]) for n0 in range(0, N, TB)] if tiled else [(0, N, None)]

        def in_gemm(src, layer, n0, nb, st):
            with _Stage("lstm_in_gemm", events, st):
                native.gemm(src[n0 * T * H:], H, layer["wih"], layer["bias"], b["gx"][n0 * T * 4 * H:], 4 * H, T * nb, 4 * H,
                            H, impl=gemm_impl, stream=st)

        self._stem(x, b, events, feats)
        if tiled:
            b["start"].record()
        for n0, nb, st in tiles:    # every tile's conv GEMM and first input GEMM are enqueued ahead of any recurrence
            if tiled:
                st.wait_event(b["start"])
            self._conv_gemm(b, n0, nb, b["ya"][n0 * T * H:], events, gemm_impl, st, stride_inner=nb)
            if feats is not None:
                feats["conv"] = b["ya"].view(T, N, H).clone()
            in_gemm(b["ya"], self.lstm[0], n0, nb, st)
        cur, nxt = b["ya"], b["yb"]
        for li, layer in enumerate(self.lstm):
            for n0, nb, st in tiles:
                if li > 0:
                    in_gemm(cur, layer, n0, nb, st)
                with _Stage("lstm_rec", events, st):
                    native.lstm_rec(b["gx"][n0 * T * 4 * H:], layer["whh"], nxt[n0 * T * H:], T, nb, H, layer["reverse"],
                                    stream=st)
            cur, nxt = nxt, cur
            if feats is not None:
                feats[f"lstm{li}"] = cur.view(T, N, H).clone()
        for i, (n0, nb, st) in enumerate(tiles):
            with _Stage("crf_gemm", events, st):    # rows r = t*nb + i_chunk -> out[n0 + i_chunk][t]
                native.gemm(cur[n0 * T * H:], H, self.wl, self.bl, out[n0:], self.n_scores, T * nb, self.n_scores, H,
                            act=self.act_l, lo=self.lo, hi=self.hi, rows_inner=nb, valid_inner=nb, stride_inner=T,
                            stride_outer=1, impl=gemm_impl, stream=st)
            if tiled:
                b["done"][i].record(st)
        if tiled:
            main = torch.cuda.current_stream()
            for done in b["done"]:
                main.wait_event(done)
        return (out, feats) if return_features else out

    # ------------------------------------------------------------------------------------------
    # tile layout (H = 384): activations [tile][T][64][H], gate pre-activations [tile][T][8][64][192]
    # ------------------------------------------------------------------------------------------
    def _plan_struct(self, b, N, L):
        """`b200_lstm_crf_plan` for this geometry and buffer set (cached in the buffer dict)."""
        if "struct" not in b:
            p = native.LstmCrfPlanStruct()
            p.n, p.l, p.t, p.tp = N, L, b["T"], b["Tp"]
            p.c1, _, p.k1 = self.w1.shape
            p.c2, _, p.k2 = self.w2.shape
            p.act1, p.act2 = self.act1, self.act2
            p.hidden, p.k3, p.s3, p.pad3, p.act3 = self.hidden, self.k3, self.s3, self.pad3, self.act3
            p.n_lstm, p.n_scores, p.act_l, p.lo, p.hi = len(self.lstm), self.n_scores, self.act_l, self.lo, self.hi
            ptr = lambda t: None if t is None else t.data_ptr()
            p.w1, p.b1, p.w2, p.b2, p.w3, p.b3 = ptr(self.w1), ptr(self.b1), ptr(self.w2), ptr(self.b2), ptr(self.w3), ptr(self.b3)
            p.wl, p.bl = ptr(self.wl), ptr(self.bl)
            for i, layer in enumerate(self.lstm):
                p.reverse[i] = int(layer["reverse"])
                p.wih[i], p.bias[i], p.whh[i] = ptr(layer["wih"]), ptr(layer["bias"]), ptr(layer["whh"])
            p.stem, p.ya, p.yb, p.gx, p.hx = (ptr(b[k]) for k in ("stem", "ya", "yb", "gx", "hx"))
            for i, st in enumerate(b["chains"]):
                p.chain_streams[i] = st.cuda_stream
            b["struct"] = p
        return b["struct"]

    def forward_tiles(self, x, out=None, gemm_impl=native.GEMM_AUTO, events=None, return_features=False, slot=0):
        """
        Forward in the tile layout: the fused LSTM kernel over the whole stack in chains of tiles, each chain on a stream of
        its own (b200_lstm_crf_lstm_fwd), or layer by layer on the current stream the int8 input-projection GEMM and the
        recurrent kernel under `quantize`.  `slot` selects one of several independent buffer sets (batches in flight at
        the same time), each with its own chain streams.
        """
        x = self._input(x)
        N, L = x.shape
        H, TB, CS = self.hidden, self.tile, self.tile_cs
        CW = 4 * H // CS                     # gx columns per cluster rank (192)
        b = self._buffers("tile", N, L, slot)
        T, nt = b["T"], b["nt"]
        if out is None:
            out = torch.empty(N, T, self.n_scores, dtype=torch.float16, device=self.device)
        if events is None and not return_features and gemm_impl == native.GEMM_AUTO and not self.quantize \
                and len(self.lstm) <= native.MAX_LSTM_LAYERS:
            # the whole encoder from ONE C-ABI call (b200_lstm_crf_fwd); the per-kernel path below runs the same launches
            # one ctypes call at a time (used when per-kernel events or intermediate activations are wanted)
            native.lstm_crf_fwd(self._plan_struct(b, N, L), x, out)
            return out

        def gather(buf):            # [tile][T][64][H] -> [T][N][H]
            return buf.permute(1, 0, 2, 3).reshape(T, nt * TB, H)[:, :N].clone()

        feats = {} if return_features else None
        self._stem(x, b, events, feats)
        # all tiles in one launch: chunk n of the stem -> (tile n / TB, row n % TB)
        self._conv_gemm(b, 0, N, b["ya"], events, gemm_impl, stride_inner=TB, group=TB, stride_group=T * TB)
        cur, nxt = b["ya"], b["yb"]
        if feats is not None:
            feats["conv"] = gather(cur)
        rows = dict(rows_inner=TB, valid_inner=TB, stride_inner=1, stride_outer=CS * TB, cb_width=CW, cb_rows=TB)
        if self.quantize:
            for li, layer in enumerate(self.lstm):
                # rows (tile, t, chunk) -> gx[tile][t][rank][chunk][CW]
                with _Stage("quantize_i8", events):
                    native.quantize_i8(cur, b["yq"], 127.0)
                with _Stage("lstm_in_gemm", events):
                    native.gemm_i8(b["yq"], H, layer["wih_q"], layer["wih_scale"], layer["bias"], b["gx"], CW, nt * T * TB,
                                   4 * H, H, **rows)
                with _Stage("lstm_rec", events):
                    native.lstm_rec_tile(b["gx"], layer["whh"], nxt, T, N, H, layer["reverse"], workspace=b["hx"])
                cur, nxt = nxt, cur
                if feats is not None:
                    feats[f"lstm{li}"] = gather(cur)
        else:
            # the stack as b200_lstm_crf_fwd runs it (chains of tiles on the slot's chain streams); layer by layer when the
            # activations between layers are wanted
            n = len(self.lstm)
            for first, count in ([(i, 1) for i in range(n)] if feats is not None else [(0, n)]):
                with _Stage("lstm_rec", events):
                    native.lstm_crf_lstm_fwd(self._plan_struct(b, N, L), first, count)
                if feats is not None:
                    feats[f"lstm{first}"] = gather(b["ya"] if first % 2 else b["yb"])
            cur = b["yb"] if n % 2 else b["ya"]
        # full tiles in one launch: rows r = (tile*T + t)*TB + i -> out[tile*TB + i][t]; a last tile the batch does not fill
        # in a launch of its own, whose `valid_inner` cuts off the rows of chunks beyond the batch
        full = N // TB
        if full:
            with _Stage("crf_gemm", events):
                native.gemm(cur, H, self.wl, self.bl, out, self.n_scores, full * T * TB, self.n_scores, H, act=self.act_l,
                            lo=self.lo, hi=self.hi, rows_inner=TB, valid_inner=TB, stride_inner=T, stride_outer=1,
                            group=T, stride_group=TB * T, impl=gemm_impl)
        if N % TB:
            with _Stage("crf_gemm", events):
                native.gemm(cur[full], H, self.wl, self.bl, out[full * TB:], self.n_scores, T * TB, self.n_scores, H,
                            act=self.act_l, lo=self.lo, hi=self.hi, rows_inner=TB, valid_inner=N - full * TB,
                            stride_inner=T, stride_outer=1, impl=gemm_impl)
        return (out, feats) if return_features else out

    # ------------------------------------------------------------------------------------------
    # wide layout (H = 768, 1024): activations [T][N][H], gate pre-activations [T][G][N][32], one grid-wide recurrent launch
    # ------------------------------------------------------------------------------------------
    def _check_wide_status(self):
        """Raise if a recurrent launch of the previous wide-path forward gave up waiting for its peer CTAs."""
        pending, self._wide_pending = self._wide_pending, None
        if pending is not None:
            done, status = pending
            done.synchronize()
            if int(status.max()) != 0:
                raise native.NativeError(
                    f"b200_lstm_rec_wide_fwd: the CTAs of the recurrent kernel stopped waiting for each other (status "
                    f"{status.tolist()} per layer); the scores of the previous batch are invalid")

    def forward_wide(self, x, out=None, gemm_impl=native.GEMM_AUTO, events=None, return_features=False):
        """
        Forward of the wide widths, layer by layer on the current stream: stem -> conv GEMM -> n_lstm x (input GEMM +
        grid-wide recurrent launch) -> CRF GEMM.  The status words of the recurrent launches are copied to pinned memory at
        the end and checked at the start of the next call (`_check_wide_status`).  Batches larger than one launch takes
        (b200_lstm_wide_max_chunks) run as consecutive sub-batches.
        """
        self._check_wide_status()
        x = self._input(x)
        N, L = x.shape
        H, G = self.hidden, self.wide
        CW = 4 * H // G                     # gx columns per CTA (32)
        cap = native.lstm_wide_max_chunks(H)
        if N > cap:
            if return_features:
                raise ValueError(f"return_features needs a batch of at most {cap} chunks at hidden size {H}")
            if out is None:
                out = torch.empty(N, self.frames(L), self.n_scores, dtype=torch.float16, device=self.device)
            for n0 in range(0, N, cap):
                self.forward_wide(x[n0:n0 + cap], out=out[n0:n0 + cap], gemm_impl=gemm_impl, events=events)
            return out
        b = self._buffers("wide", N, L)
        T = b["T"]
        feats = {} if return_features else None

        def stage(name):
            return _Stage(name, events)

        self._stem(x, b, events, feats)
        cur, nxt = b["ya"], b["yb"]
        self._conv_gemm(b, 0, N, cur, events, gemm_impl, stride_inner=N)
        if feats is not None:
            feats["conv"] = cur.clone()
        for i, layer in enumerate(self.lstm):
            with stage("lstm_in_gemm"):     # rows r = t*N + n -> gx[t][g][n][:], column block g = units [8g, 8g + 8)
                native.gemm(cur, H, layer["wih"], layer["bias"], b["gx"], CW, T * N, 4 * H, H, rows_inner=N, valid_inner=N,
                            stride_inner=1, stride_outer=G * N, cb_width=CW, cb_rows=N, impl=gemm_impl)
            with stage("lstm_rec"):
                native.lstm_rec_wide(b["gx"], layer["whh"], nxt, T, N, H, layer["reverse"], workspace=b["ws"])
            b["status"][i:i + 1].copy_(b["ws_status"])
            cur, nxt = nxt, cur
            if feats is not None:
                feats[f"lstm{i}"] = cur.clone()
        if self.wb is not None:
            with stage("bottleneck_gemm"):  # rows r = t*N + n -> yl[t][n][:]
                native.gemm(cur, H, self.wb, self.bb, b["yl"], self.head_in, T * N, self.head_in, H, impl=gemm_impl)
            cur = b["yl"]
            if feats is not None:
                feats["linear"] = cur.clone()

        if out is None:
            out = torch.empty(N, T, self.n_scores, dtype=torch.float16, device=self.device)
        with stage("crf_gemm"):             # rows r = t*N + n -> out[n][t][:]
            native.gemm(cur, self.head_in, self.wl, self.bl, out, self.n_scores, T * N, self.n_scores, self.head_in,
                        act=self.act_l, lo=self.lo, hi=self.hi,
                        rows_inner=N, valid_inner=N, stride_inner=T, stride_outer=1, impl=gemm_impl)
        status = torch.empty(len(self.lstm), dtype=torch.int32, pin_memory=True)
        status.copy_(b["status"], non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        self._wide_pending = (done, status)
        return (out, feats) if return_features else out

    # ------------------------------------------------------------------------------------------
    def forward(self, x, out=None, gemm_impl=native.GEMM_AUTO, return_features=False, events=None, tiled=None, slot=0):
        """
        x: [N, 1, L] (or [N, L]) fp16 CUDA -> scores [N, T, C] fp16 (no blank column); with `return_features`, the pair
        (scores, dict of intermediate activations).
        `events`: optional list; (stage, start, end) CUDA events are appended per kernel.
        `tiled`: the schedule of the generic layout (see `forward_generic`); the tile and wide layouts have one schedule
        each and ignore it.
        `slot`: the buffer set of the tile layout (see `forward_tiles`); the other layouts have only slot 0.
        """
        with torch.cuda.device(self.device):    # streams / events / launches belong to the plan's device, whatever is current
            if self.supports_slots:
                return self.forward_tiles(x, out=out, gemm_impl=gemm_impl, events=events, return_features=return_features,
                                          slot=slot)
            if slot != 0:
                raise NotImplementedError("several batches in flight (slot != 0) need the tile-layout path (hidden size 384)")
            if self.wide:
                return self.forward_wide(x, out=out, gemm_impl=gemm_impl, events=events, return_features=return_features)
            return self.forward_generic(x, out=out, gemm_impl=gemm_impl, events=events, return_features=return_features,
                                        tiled=tiled)


class _LazyStreams:
    """Per-tile streams of the generic layout, created on first use with `native.new_stream` (CUDA streams of their
    own).  `torch.cuda.Stream()` hands out streams from a pool of 32 per device round-robin: the 22 per-tile streams of two buffer
    sets, created eagerly, pushed later requests (the slot and copy streams of `score_batches`) onto pool entries already in use
    -- two "different" streams were then one CUDA stream and batches meant to overlap ran back to back (end-to-end step 17 ->
    20-58 ms, depending on how many streams the process had created before)."""

    def __init__(self, device, n):
        self.device, self.items = device, [None] * n

    def __getitem__(self, i):
        if self.items[i] is None:
            self.items[i] = native.new_stream(self.device)
        return self.items[i]

    def __len__(self):
        return len(self.items)


def compile_lstm_crf(encoder, device, quantize=False):
    return LstmCrfPlan(encoder, device, quantize=quantize)


def score_layout(width, state_len=None):
    """(state_len, learned_blank) of CRF scores `width` columns wide: 4**(k+1) = moves only, the fixed-blank layout
    [state][m0..m3]; 5 * 4**k = learned blanks, the CTC_CRF layout [state][stay, m0..m3].  The two never coincide.
    `state_len`: the model's, checked against the width; None: inferred from it."""
    for k in ((state_len,) if state_len is not None else range(1, 9)):
        if width == 4 ** (k + 1):
            return k, False
        if width == 5 * 4 ** k:
            return k, True
    raise ValueError(f"scores width {width} is neither 4**(k+1) (fixed blank) nor 5 * 4**k (learned blank)"
                     + ("" if state_len is None else f" for state_len {state_len}"))


class CrfDecoder:
    """Workspace-caching wrapper around b200_crf_decode (fixed blank: scores [N, T, 4**(k+1)], [state][m0..m3]) and
    b200_crf_decode_lb (learned blank: scores [N, T, 5 * 4**k], [state][stay, m0..m3]); the score width picks the kernel."""

    def __init__(self):
        self._ws_by_device = {}     # one workspace per (device, host thread): basecall() decodes on background threads

    def __call__(self, scores, state_len, blank_score=2.0, qscale=1.0, qbias=0.0, events=None, out=None, slot=0, beam=None):
        """`beam=(beam_width, beam_cut)`: run the beam search (after the forward-backward pass) instead of the exact
        posterior-Viterbi trace-back (fixed blank only).  `blank_score` is ignored for learned-blank scores."""
        with torch.cuda.device(scores.device):
            return self._call(scores, state_len, blank_score, qscale, qbias, events, out, slot, beam)

    def _call(self, scores, state_len, blank_score, qscale, qbias, events, out, slot=0, beam=None):
        """-> (moves, sequence, qstring) uint8 [N, T] on the device; `out`: optional uint8 [3, N, T] to write them into."""
        n, t, c = scores.shape
        _, learned = score_layout(c, state_len)
        if learned and beam is not None:
            raise ValueError("the beam search kernel needs a fixed blank score; scores with learned blank scores "
                             "(5 * 4**state_len columns) decode with the exact decoder only")
        scores = scores.to(torch.float16).contiguous()
        need = native.crf_decode_workspace_bytes(n, t, state_len)
        key = (scores.device, threading.get_ident(), slot)
        ws = self._ws_by_device.get(key)
        if ws is None or ws.numel() < need:
            ws = self._ws_by_device[key] = torch.empty(need, dtype=torch.uint8, device=scores.device)
        outs = list(out) if out is not None else [torch.empty(n, t, dtype=torch.uint8, device=scores.device) for _ in range(3)]
        with _Stage("crf_decode", events):
            if learned:
                native.crf_decode_lb(scores, state_len, qscale, qbias, ws, *outs)
            elif beam is None:
                native.crf_decode(scores, state_len, blank_score, qscale, qbias, ws, *outs)
            else:
                native.crf_beam_search(scores, state_len, blank_score, beam[0], beam[1], qscale, qbias, ws, *outs)
        return tuple(outs)  # moves, sequence, qstring
