"""
Functional re-statement of the QuartzNet module tree (bonito_b200/ctc/model.py, reference bonito/ctc/model.py) in train
mode, with the dropout masks as inputs, for the training tests.

`forward(model, x, masks, dtype, device, autocast)` runs the blocks with F.conv1d and F.batch_norm(training=True) on leaf
copies of the model's parameters (float64 on the CPU for the oracle; fp32 master copies under fp16 autocast on the GPU for
torch's own gradients) and copies of the running statistics, which F.batch_norm updates.  masks[u] is the keep mask (bool
[N, C, T]) of the u-th activation in module order, or None for p = 0; a kept element is scaled by 1 / (1 - p).
"""

import torch
import torch.nn.functional as F

from bonito_b200.ctc.model import TCSConv1d


def _units(model):
    """(block, [(TCSConv1d, BatchNorm1d)], p) per block."""
    out = []
    for blk in model.encoder.encoder:
        mods = [m for m in blk.conv if isinstance(m, (TCSConv1d, torch.nn.BatchNorm1d))]
        p = blk.activation[1].p
        out.append((blk, list(zip(mods[0::2], mods[1::2])), p))
    return out


def forward(model, x, masks, dtype=torch.float64, device="cpu", autocast=False):
    """-> (log-probs [N, T, 5], {parameter name: leaf tensor}, {buffer name: updated running statistic})."""
    names = {id(p): n for n, p in model.named_parameters()}
    bnames = {id(b): n for n, b in model.named_buffers()}
    P = {n: p.detach().to(device=device, dtype=dtype).clone().requires_grad_(True) for n, p in model.named_parameters()}
    B = {n: b.detach().to(device=device, dtype=dtype if b.is_floating_point() else b.dtype).clone()
         for n, b in model.named_buffers()}
    act = model.encoder.encoder[0].activation[0]
    unit = [0]

    def conv(c, h):
        return F.conv1d(h, P[names[id(c.weight)]], None, c.stride, c.padding, c.dilation, c.groups)

    def tcs(t, h):
        return conv(t.pointwise, conv(t.depthwise, h)) if t.separable else conv(t.conv, h)

    def bn(b, z):
        return F.batch_norm(z, B[bnames[id(b.running_mean)]], B[bnames[id(b.running_var)]], P[names[id(b.weight)]],
                            P[names[id(b.bias)]], training=True, momentum=b.momentum, eps=b.eps)

    def act_drop(v, p):
        v = act(v)
        m = masks[unit[0]]
        unit[0] += 1
        if p > 0:
            v = v * m.to(device) * (1.0 / (1.0 - p))
        return v

    with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
        h = x.to(device=device, dtype=dtype)
        if h.dim() == 2:
            h = h[:, None, :]
        for blk, pairs, p in _units(model):
            hin = h
            for r, (t, b) in enumerate(pairs):
                z = bn(b, tcs(t, h))
                if r < len(pairs) - 1:
                    h = act_drop(z, p)
            if blk.use_res:
                res = blk.residual
                z = z + bn(res[1], conv(res[0].conv, hin))
            h = act_drop(z, p)
        head = model.decoder.layers[0]
        logits = F.conv1d(h, P[names[id(head.weight)]], P[names[id(head.bias)]])
        logp = F.log_softmax(logits.permute(0, 2, 1), dim=-1)
    for b in model.modules():
        if isinstance(b, torch.nn.BatchNorm1d):
            B[bnames[id(b.num_batches_tracked)]] += 1
    return logp, P, B


def loss(logp, targets, lengths):
    """Model.loss on [N, T, C] log-probs in their own dtype and device: CTC (mean) + the default label smoothing."""
    lp = logp.permute(1, 0, 2).float() if logp.dtype != torch.float64 else logp.permute(1, 0, 2)
    T, N, C = lp.shape
    weights = torch.cat([torch.tensor([0.4]), (0.1 / (C - 1)) * torch.ones(C - 1)]).to(lp)
    il = torch.full((N,), T, dtype=torch.int64)
    ctc = F.ctc_loss(lp, targets.to(lp.device), il, lengths, reduction="mean")
    return ctc - (lp * weights).mean()


def unpack_masks(bits, N, T, C):
    """keep bits [N*T, C/8] uint8 (bit j of byte b: channel 8b + j) -> bool [N, C, T]."""
    b = bits.to(torch.int64)
    keep = ((b[:, :, None] >> torch.arange(8, device=bits.device)) & 1).bool().reshape(N * T, C)
    return keep.view(N, T, C).permute(0, 2, 1).contiguous()
