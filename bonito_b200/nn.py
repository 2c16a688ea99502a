"""
Layer registry for bonito_b200 -- the host-side mirror of `bonito.nn`.

This module keeps the reference's plugin surface for the chunked forward path
(`bonito/nn.py:13-19` registry, `:418-444` to_dict/from_dict,
`:447-454` fuse_bn_) so that model `config.toml` files written for the reference
build the same module tree here, with the same `state_dict()` key names and
shapes (`match_names`, `bonito/util.py:239-248`, pairs
checkpoints to modules by sorted shape).

The torch modules in this file are *descriptions plus parameter storage*: the
native engine (`bonito_b200.engine`) walks the tree, packs the weights and runs
the hand-written sm_90a kernels.  `forward()` on the individual layers is a
plain-torch definition of the layer semantics, used on CPU by the host-logic
tests; it is never the product path on a GPU box (see `bonito_b200.crf.model`).
"""

from collections import OrderedDict

import torch
from torch import nn as tnn

Module = tnn.Module

#: name -> layer class; populated by `register` (reference: bonito/nn.py:13).
layers = {}


def register(layer):
    """Class decorator: publish `layer` under its lower-cased class name."""
    layer.name = layer.__name__.lower()
    layers[layer.name] = layer
    return layer


def _activation(spec):
    """Resolve an activation spec (registry name, None, or a ready module)."""
    if spec in layers:
        return layers[spec]()
    return spec


def _described(layer, include_weights=False):
    return layer.to_dict(include_weights) if hasattr(layer, "to_dict") else {}


def to_dict(layer, include_weights=False):
    """Serialise a layer into the TOML-style dict `from_dict` understands."""
    return {"type": layer.name, **_described(layer, include_weights)}


def from_dict(model_dict, layer_types=None):
    """
    Build a module tree from a nested dict (reference: bonito/nn.py:424-444).

    * non-dicts pass through untouched (already-built objects);
    * `type` selects the class from `layer_types` (default: the registry);
    * a class-level `from_dict` takes over construction when present;
    * `sublayers` may be a list of dicts or a single dict;
    * every other key is a constructor kwarg; constructor failures are re-raised
      with the layer type and arguments in the message.
    """
    if not isinstance(model_dict, dict):
        return model_dict
    spec = dict(model_dict)
    table = layers if layer_types is None else layer_types
    cls = table[spec.pop("type")]
    if hasattr(cls, "from_dict"):
        return cls.from_dict(spec, table)
    if "sublayers" in spec:
        sub = spec["sublayers"]
        if isinstance(sub, list):
            spec["sublayers"] = [from_dict(s, table) for s in sub]
        else:
            spec["sublayers"] = from_dict(sub, table)
    try:
        return cls(**spec)
    except Exception as err:
        raise Exception(f"Failed to build layer of type {cls} with args {spec}") from err


register(tnn.ReLU)
register(tnn.Tanh)


@register
class Swish(tnn.SiLU):
    """x * sigmoid(x)."""


@register
class Linear(Module):
    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.in_features, self.out_features, self.bias = in_features, out_features, bias
        self.linear = tnn.Linear(in_features, out_features, bias=bias)

    def forward(self, x):
        return self.linear(x)

    def to_dict(self, include_weights=False):
        out = dict(in_features=self.in_features, out_features=self.out_features, bias=self.bias)
        if include_weights:
            out["params"] = {"W": self.linear.weight,
                             "b": self.linear.bias if self.bias is not None else []}
        return out


@register
class Clamp(Module):
    def __init__(self, min, max):
        super().__init__()
        self.min, self.max = min, max

    def forward(self, x):
        return x.clamp(self.min, self.max)

    def to_dict(self, include_weights=False):
        return {"min": self.min, "max": self.max}


@register
class Serial(tnn.Sequential):
    def __init__(self, sublayers):
        super().__init__(*sublayers)

    def forward(self, x, return_features=False):
        if not return_features:
            return super().forward(x)
        feats = []
        for layer in self:
            x = layer(x)
            feats.append(x)
        return x, feats

    def to_dict(self, include_weights=False):
        return {"sublayers": [to_dict(m, include_weights) for m in self._modules.values()]}

    def __repr__(self):
        return tnn.ModuleList.__repr__(self)


@register
class Stack(Serial):
    """`depth` independent copies of one layer description."""

    @classmethod
    def from_dict(cls, model_dict, layer_types=None):
        return cls([from_dict(model_dict["layer"], layer_types) for _ in range(model_dict["depth"])])

    def to_dict(self, include_weights=False):
        if include_weights:
            raise NotImplementedError
        descr = [to_dict(m) for m in self]
        assert all(d == descr[0] for d in descr[1:]), "all layers should be the same"
        return {"layer": descr[0], "depth": len(self)}


@register
class NamedSerial(tnn.Sequential):
    @classmethod
    def from_dict(cls, model_dict, layer_types=None):
        return cls({name: from_dict(spec, layer_types) for name, spec in model_dict.items()})

    def __init__(self, layers):
        super().__init__(OrderedDict(layers.items()))

    def to_dict(self, include_weights=False):
        if include_weights:
            raise NotImplementedError
        return {name: to_dict(m) for name, m in self.named_children()}


class MakeContiguous(Module):
    def forward(self, x):
        return x.contiguous()


@register
class LinearUpsample(Module):
    """Linear d_model -> scale_factor*d_model, then fold the factor into time."""

    def __init__(self, d_model, scale_factor, batch_first=True):
        super().__init__()
        self.d_model, self.scale_factor, self.batch_first = d_model, scale_factor, batch_first
        self.linear = tnn.Linear(d_model, scale_factor * d_model)

    def forward(self, src):
        if not self.batch_first:
            src = src.permute(1, 0, 2)
        n, length, width = src.shape
        out = self.linear(src).reshape(n, self.scale_factor * length, width)
        return out if self.batch_first else out.permute(1, 0, 2)

    def output_stride(self, input_stride):
        return input_stride // self.scale_factor

    def to_dict(self, include_weights=False):
        if include_weights:
            raise NotImplementedError
        return dict(d_model=self.d_model, scale_factor=self.scale_factor, batch_first=self.batch_first)


@register
class Reverse(Module):
    def __init__(self, sublayers):
        super().__init__()
        self.layer = Serial(sublayers) if isinstance(sublayers, list) else sublayers

    def forward(self, x):
        return self.layer(x.flip(0)).flip(0)

    def to_dict(self, include_weights=False):
        if isinstance(self.layer, Serial):
            return self.layer.to_dict(include_weights)
        return {"sublayers": to_dict(self.layer, include_weights)}


@register
class BatchNorm(Module):
    def __init__(self, num_features, eps=1e-05, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        self.bn = tnn.BatchNorm1d(num_features, eps, momentum, affine, track_running_stats)

    def forward(self, x):
        return self.bn(x)

    def to_dict(self, include_weights=False):
        bn = self.bn
        out = dict(num_features=bn.num_features, eps=bn.eps, momentum=bn.momentum,
                   affine=bn.affine, track_running_stats=bn.track_running_stats)
        if include_weights:
            params = {}
            if bn.affine:
                params.update(W=bn.weight, b=bn.bias)
            if bn.track_running_stats:
                params.update(running_mean=bn.running_mean, running_var=bn.running_var)
            out["params"] = params
        return out


@register
class Convolution(Module):
    """Conv1d -> optional norm -> optional activation (reference: bonito/nn.py:221-241)."""

    def __init__(self, insize, size, winlen, stride=1, padding=0, bias=True, activation=None, norm=None):
        super().__init__()
        self.conv = tnn.Conv1d(insize, size, winlen, stride=stride, padding=padding, bias=bias)
        self.activation = _activation(activation)
        if isinstance(norm, dict):
            norm = from_dict(norm)
        elif isinstance(norm, str):
            norm = layers[norm](size)
        self.norm = norm

    def forward(self, x):
        y = self.conv(x)
        if self.norm is not None:
            y = self.norm(y)
        return y if self.activation is None else self.activation(y)

    def to_dict(self, include_weights=False):
        c = self.conv
        out = dict(insize=c.in_channels, size=c.out_channels, bias=c.bias is not None,
                   winlen=c.kernel_size[0], stride=c.stride[0], padding=c.padding[0])
        if self.activation is not None:
            out["activation"] = self.activation.name
        if self.norm is not None:
            out["norm"] = to_dict(self.norm, include_weights)
            if not include_weights and self.norm.name in layers:
                # collapse a default-constructed norm back to its registry name
                if out["norm"] == to_dict(layers[self.norm.name](out["size"])):
                    out["norm"] = self.norm.name
        if include_weights:
            out["params"] = {"W": c.weight, "b": c.bias if c.bias is not None else []}
        return out


@register
class LinearCRFEncoder(Module):
    """
    Linear -> [activation] -> [*scale] -> [insert fixed blank column].

    Output width is n_base**(state_len+1) when `blank_score` is fixed, else
    (n_base+1)*n_base**state_len (reference: bonito/nn.py:268-298).
    """

    def __init__(self, insize, n_base, state_len, bias=True, scale=None, activation=None,
                 blank_score=None, expand_blanks=True, permute=None):
        super().__init__()
        self.n_base, self.state_len = n_base, state_len
        self.scale, self.blank_score, self.expand_blanks, self.permute = scale, blank_score, expand_blanks, permute
        width = n_base ** (state_len + 1) if blank_score is not None else (n_base + 1) * n_base ** state_len
        self.linear = tnn.Linear(insize, width, bias=bias)
        self.activation = _activation(activation)

    def forward(self, x):
        if self.permute is not None:
            x = x.permute(*self.permute)
        s = self.linear(x)
        if self.activation is not None:
            s = self.activation(s)
        if self.scale is not None:
            s = s * self.scale
        if self.blank_score is not None and self.expand_blanks:
            t, n, c = s.shape
            s = torch.nn.functional.pad(
                s.view(t, n, c // self.n_base, self.n_base), (1, 0, 0, 0, 0, 0, 0, 0), value=self.blank_score
            ).view(t, n, -1)
        return s

    def to_dict(self, include_weights=False):
        out = dict(insize=self.linear.in_features, n_base=self.n_base, state_len=self.state_len,
                   bias=self.linear.bias is not None, scale=self.scale,
                   blank_score=self.blank_score, expand_blanks=self.expand_blanks)
        if self.activation is not None:
            out["activation"] = self.activation.name
        if self.permute is not None:
            out["permute"] = self.permute
        if include_weights:
            out["params"] = {"W": self.linear.weight,
                             "b": self.linear.bias if self.linear.bias is not None else []}
        return out

    def extra_repr(self):
        text = f"n_base={self.n_base}, state_len={self.state_len}, scale={self.scale}, " \
               f"blank_score={self.blank_score}, expand_blanks={self.expand_blanks}"
        return text + (f", permute={self.permute}" if self.permute else "")


@register
class Permute(Module):
    def __init__(self, dims):
        super().__init__()
        self.dims = dims

    def forward(self, x):
        return x.permute(*self.dims)

    def to_dict(self, include_weights=False):
        return {"dims": self.dims}

    def extra_repr(self):
        return f"dims={self.dims}"


def truncated_normal(size, dtype=torch.float32, device=None, num_resample=5):
    """Standard normal resampled (up to `num_resample` draws) into (-2, 2)."""
    draws = torch.empty(tuple(size) + (num_resample,), dtype=torch.float32, device=device).normal_()
    first_ok = ((draws < 2) & (draws > -2)).max(-1, keepdim=True)[1]
    return draws.gather(-1, first_ok).squeeze(-1).clamp_(-2, 2)


class RNNWrapper(Module):
    """
    One unidirectional torch RNN layer with an optional time flip
    (reference: bonito/nn.py:353-400).  The state bias `bias_hh` is frozen at 0.
    """

    def __init__(self, rnn_type, *args, reverse=False, orthogonal_weight_init=True,
                 disable_state_bias=True, bidirectional=False, **kwargs):
        super().__init__()
        if reverse and bidirectional:
            raise Exception("'reverse' and 'bidirectional' should not both be set to True")
        self.reverse = reverse
        self.rnn = rnn_type(*args, bidirectional=bidirectional, **kwargs)
        self.init_orthogonal(orthogonal_weight_init)
        self.init_biases()
        if disable_state_bias:
            self.disable_state_bias()

    def forward(self, x):
        if self.reverse:
            x = x.flip(0)
        y, _ = self.rnn(x)
        return y.flip(0) if self.reverse else y

    def init_biases(self, types=("bias_ih",)):
        with torch.no_grad():
            for name, p in self.rnn.named_parameters():
                if any(t in name for t in types):
                    p.copy_(0.5 * truncated_normal(p.shape, dtype=p.dtype, device=p.device))

    def init_orthogonal(self, types=True):
        if not types:
            return
        if types is True:
            types = ("weight_ih", "weight_hh")
        h = self.rnn.hidden_size
        for name, p in self.rnn.named_parameters():
            if any(t in name for t in types):
                for row in range(0, p.size(0), h):
                    tnn.init.orthogonal_(p[row:row + h])

    def disable_state_bias(self):
        for name, p in self.rnn.named_parameters():
            if "bias_hh" in name:
                p.requires_grad = False
                p.zero_()

    def extra_repr(self):
        return f"reverse={bool(self.reverse)}"


@register
class LSTM(RNNWrapper):
    def __init__(self, size, insize, bias=True, reverse=False):
        super().__init__(tnn.LSTM, insize, size, bias=bias, reverse=reverse)

    def to_dict(self, include_weights=False):
        r = self.rnn
        out = dict(size=r.hidden_size, insize=r.input_size, bias=r.bias, reverse=self.reverse)
        if include_weights:
            out["params"] = {"iW": r.weight_ih_l0.reshape(4, r.hidden_size, r.input_size),
                             "sW": r.weight_hh_l0.reshape(4, r.hidden_size, r.hidden_size),
                             "b": r.bias_ih_l0.reshape(4, r.hidden_size)}
        return out


def fuse_bn_(m):
    """Put `m` in eval mode; fold a Convolution's BatchNorm into its Conv1d."""
    m.training = False
    if isinstance(m, Convolution) and isinstance(m.norm, BatchNorm):
        m.conv = tnn.utils.fusion.fuse_conv_bn_eval(m.conv, m.norm.bn)
        m.norm = None
