"""Feature trunks: MLPBase and CNNBase (API of /root/reference/torchrl/networks/base.py:8-107).

Plain ``nn.Module``s -- the north star keeps the small policy/value nets in PyTorch (cuBLAS);
everything around them is in the CUDA library.
"""
import numpy as np
import torch
import torch.nn as nn

from . import init as winit
from . import fused


class MLPBase(nn.Module):
    """Linear -> act, repeated; the last hidden layer keeps an activation too
    (`last_activation_func`, defaulting to `activation_func`; base.py:24-41)."""

    def __init__(self, input_shape, hidden_shapes, activation_func=nn.ReLU, init_func=winit.basic_init,
                 add_ln=False, last_activation_func=None):
        super().__init__()
        self.activation_func = activation_func
        self.add_ln = add_ln
        self.last_activation_func = last_activation_func if last_activation_func is not None else activation_func
        width = int(np.prod(input_shape))
        self.output_shape = width
        layers = []
        for i, h in enumerate(hidden_shapes):
            fc = nn.Linear(width, h)
            init_func(fc)
            layers.append(fc)
            last = (i == len(hidden_shapes) - 1)
            if last and not add_ln:
                layers.append(self.last_activation_func())
            else:
                layers.append(activation_func())
                if add_ln:
                    layers.append(nn.LayerNorm(h))
            width = h
            self.output_shape = h
        if add_ln and layers:
            # reference quirk (base.py:39-40): the trailing LayerNorm is dropped and replaced by
            # the last activation
            layers.pop(-1)
            layers.append(self.last_activation_func())
        self.fcs = layers
        self.seq_fcs = nn.Sequential(*layers)
        # (Linear, activation) pairs eligible for the fused CUDA epilogue (no LayerNorm in between)
        self._pairs = None
        if not add_ln and len(layers) % 2 == 0 and all(isinstance(layers[i], nn.Linear) for i in range(0, len(layers), 2)):
            self._pairs = [(layers[i], layers[i + 1]) for i in range(0, len(layers), 2)]

    def forward(self, x):
        if self._pairs and fused.fused_enabled() and x.is_cuda:
            for fc, act in self._pairs:
                x = self._pair(x, fc, act)
            return x
        return self.seq_fcs(x)

    @staticmethod
    def _pair(x, fc, act):
        if fused.can_fuse(x, fc, act):
            return fused.linear_act(x, fc, fused.ACT_CODES[type(act)])
        return act(fc(x))

    def forward_with_head(self, x, head):
        """head(self(x)) with the last hidden layer and the output layer as one fused autograd node when the
        shapes allow (fused._MLPTail); None when they do not (the caller then takes the plain route)."""
        if not (self._pairs and fused.fused_enabled() and x.is_cuda):
            return None
        if len(self._pairs) == 2:
            (fc1, act1), (fc, act) = self._pairs
            if fused.first_ok(x, fc1, act1) and fused.tail_ok(x, fc, act, head):
                # the whole MLP as one node: the backward reduces dH1 to the first layer's gradients in place
                return fused.mlp_tail(x, fc, fused.ACT_CODES[type(act)], head,
                                      first=(fc1, fused.ACT_CODES[type(act1)]))
        for fc, act in self._pairs[:-1]:
            x = self._pair(x, fc, act)
        fc, act = self._pairs[-1]
        if not fused.tail_ok(x, fc, act, head):
            return head_plain(self._pair(x, fc, act), head)
        return fused.mlp_tail(x, fc, fused.ACT_CODES[type(act)], head)


def head_plain(h, head):
    if h.is_cuda and h.dtype == torch.float32:
        return fused.linear_plain(h, head)
    return head(h)


def calc_next_shape(input_shape, conv_info):
    out_channels, kernel_size, stride, padding = conv_info
    _, h, w = input_shape
    h = int((h + 2 * padding[0] - (kernel_size[0] - 1) - 1) / stride[0] + 1)
    w = int((w + 2 * padding[1] - (kernel_size[1] - 1) - 1) / stride[1] + 1)
    return (out_channels, h, w)


class CNNBase(nn.Module):
    """Conv stack over (..., C, H, W) inputs flattened to (..., features) (base.py:59-107)."""

    def __init__(self, input_shape, hidden_shapes, activation_func=nn.ReLU, init_func=winit.basic_init,
                 add_ln=False, last_activation_func=None):
        super().__init__()
        self.add_ln = add_ln
        self.activation_func = activation_func
        self.last_activation_func = last_activation_func if last_activation_func is not None else activation_func
        shape = tuple(input_shape)
        channels = shape[0]
        self.output_shape = shape[0] * shape[1] * shape[2]
        layers = []
        for info in hidden_shapes:
            out_c, k, s, p = info
            conv = nn.Conv2d(channels, out_c, tuple(k), tuple(s), tuple(p))
            init_func(conv)
            layers.append(conv)
            layers.append(activation_func())
            channels = out_c
            shape = calc_next_shape(shape, info)
            if add_ln:
                layers.append(nn.LayerNorm(shape[1:]))
            self.output_shape = shape[0] * shape[1] * shape[2]
        if layers:
            layers.pop(-1)
            layers.append(self.last_activation_func())
        self.convs = layers
        self.seq_convs = nn.Sequential(*layers)

    def forward(self, x):
        lead = x.shape[:-3]
        out = self.seq_convs(x.reshape((-1,) + tuple(x.shape[-3:])))
        return out.reshape(tuple(lead) + (-1,))
