"""Heads on top of a trunk: Net, FlattenNet, QNet, ZeroNet, BootstrappedNet
(API of /root/reference/torchrl/networks/nets.py:8-141)."""
import torch
import torch.nn as nn

from . import init as winit
from . import fused


class ZeroNet(nn.Module):
    def forward(self, x):
        return torch.zeros(1)


def _append_stack(in_width, hidden, out_width, act, add_ln, hidden_init, last_init):
    layers = []
    for h in hidden:
        fc = nn.Linear(in_width, h)
        hidden_init(fc)
        layers += [fc, act()]
        if add_ln:
            layers.append(nn.LayerNorm(h))
        in_width = h
    last = nn.Linear(in_width, out_width)
    last_init(last)
    layers.append(last)
    return layers


class Net(nn.Module):
    """trunk (`base_type(**kwargs)`) -> optional hidden layers -> linear output (nets.py:13-52)."""

    def __init__(self, output_shape, base_type, append_hidden_shapes=[], append_hidden_init_func=winit.basic_init,
                 net_last_init_func=winit.uniform_init, activation_func=nn.ReLU, add_ln=False, **kwargs):
        super().__init__()
        self.base = base_type(activation_func=activation_func, add_ln=add_ln, **kwargs)
        self.add_ln = add_ln
        self.activation_func = activation_func
        self.append_fcs = _append_stack(self.base.output_shape, append_hidden_shapes, output_shape, activation_func,
                                        add_ln, append_hidden_init_func, net_last_init_func)
        self.seq_append_fcs = nn.Sequential(*self.append_fcs)

    def _head(self, h):
        if (len(self.append_fcs) == 1 and fused.fused_enabled() and h.is_cuda and h.dtype == torch.float32):
            return fused.linear_plain(h, self.append_fcs[0])
        return self.seq_append_fcs(h)

    def _trunk_head(self, x):
        if len(self.append_fcs) == 1 and hasattr(self.base, "forward_with_head") and fused.fused_enabled():
            out = self.base.forward_with_head(x, self.append_fcs[0])
            if out is not None:
                return out
        return self._head(self.base(x))

    def forward(self, x):
        return self._trunk_head(x)


class FlattenNet(Net):
    def forward(self, input):
        return super().forward(torch.cat(input, dim=-1))


class QNet(Net):
    """Q(s, a): the two inputs are concatenated along the feature axis (nets.py:61-68)."""

    def forward(self, input):
        assert len(input) == 2, "Q Net only get observation and action"
        state, action = input
        return self._trunk_head(torch.cat([state, action], dim=-1))


class BootstrappedNet(nn.Module):
    """Shared trunk with `head_num` independent heads (nets.py:71-134)."""

    def __init__(self, output_shape, base_type, head_num=10, append_hidden_shapes=[],
                 append_hidden_init_func=winit.basic_init, net_last_init_func=winit.uniform_init,
                 activation_func=nn.ReLU, add_ln=False, **kwargs):
        super().__init__()
        self.base = base_type(activation_func=activation_func, add_ln=add_ln, **kwargs)
        self.add_ln = add_ln
        self.activation_func = activation_func
        self.bootstrapped_heads = nn.ModuleList()
        for _ in range(head_num):
            self.bootstrapped_heads.append(nn.Sequential(*_append_stack(
                self.base.output_shape, append_hidden_shapes, output_shape, activation_func, add_ln,
                append_hidden_init_func, net_last_init_func)))

    def forward(self, x, head_idxs):
        feature = self.base(x)
        return [self.bootstrapped_heads[i](feature) for i in head_idxs]

    def all_heads(self, x):
        """Every head on one trunk pass, as one contiguous (head_num, M, output_shape) tensor."""
        feature = self.base(x)
        return torch.stack([head(feature) for head in self.bootstrapped_heads])


class FlattenBootstrappedNet(BootstrappedNet):
    def forward(self, input, head_idxs):
        return super().forward(torch.cat(input, dim=-1), head_idxs)
