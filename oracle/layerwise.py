"""One attention layer at a time, at any floating-point precision (TEST INFRASTRUCTURE, CPU only).

`restate.forward` chains all layers in fp32, so comparing the engine with it measures the rounding of the whole network at once.
The helpers here evaluate `restate.att_layer` on a given layer input -- typically the engine's own output of the previous layer --
in float64, so a comparison measures the rounding of that one layer only.  The graph, its edge types and the global edge gate are
the ones of the fp32 oracle's trace (the engine's `edge_index` is asserted bit-exact against it elsewhere).

`restate` builds its scatter buffers with `torch.zeros(...)`, so the float64 evaluation runs under `torch.set_default_dtype`;
`default_dtype` restores the previous default in every case.
"""
import contextlib
import re

import numpy as np
import torch
import torch.nn.functional as F

from . import restate
from .synth import DEFAULT_MODEL_CONFIG

_BLOCK_KEY = re.compile(r'^refine_net\.base_block\.(\d+)\.')


@contextlib.contextmanager
def default_dtype(dtype):
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def prefix_state_dict(sd, n_layers):
    """The state dict of the same network cut after its first `n_layers` attention layers (what a ScorePosNet3D built with
    num_layers = n_layers loads strictly)."""
    out = {}
    for key, v in sd.items():
        m = _BLOCK_KEY.match(key)
        if m is None or int(m.group(1)) < n_layers:
            out[key] = v
    return out


def _cast(sd, dtype):
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}


def global_edge_weight(sd, x, edge_index, dtype=torch.float64):
    """ew_net_type='global' gate from the block's input coordinates (models/uni_transformer.py:312-318), in `dtype`."""
    sdd = _cast({k: v for k, v in sd.items() if k.startswith('refine_net.')}, dtype)
    src, dst = edge_index
    with default_dtype(dtype):
        x = x.to(dtype)
        dist = torch.norm(x[dst] - x[src], p=2, dim=-1, keepdim=True)
        dist_feat = restate.gaussian_smearing(dist, sdd['refine_net.distance_expansion.offset'])
        return torch.sigmoid(restate.mlp(sdd, 'refine_net.edge_pred_layer', dist_feat)).view(-1)


class LayerRef:
    """Attention layer l of a network (state dict `sd`, config `cfg`) on a fixed graph: `edge_index` [2,E] and `edge_type` (codes
    0..3, as `trace['edge_type']`), `mask_ligand` [N] and, for ew_net_type='global', the gate `e_w` [E] (None: computed from `x0`)."""

    def __init__(self, sd, cfg, edge_index, edge_type, mask_ligand, x0=None, e_w=None, dtype=torch.float64):
        self.cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
        self.dtype = dtype
        self.sd = _cast(sd, dtype)
        self.edge_index = edge_index
        self.edge_type = F.one_hot(edge_type.long(), num_classes=4)
        self.mask_ligand = mask_ligand
        self.e_w = None
        if self.cfg['ew_net_type'] == 'global':
            self.e_w = (e_w if e_w is not None else global_edge_weight(sd, x0, edge_index, dtype)).to(dtype)

    def __call__(self, l, h, x, fix_x=False):
        c = self.cfg
        with default_dtype(self.dtype):
            return restate.att_layer(self.sd, 'refine_net.base_block.%d' % l, h.to(self.dtype), x.to(self.dtype), self.edge_type,
                                     self.edge_index, self.mask_ligand, self.e_w, c['n_heads'], fix_x=fix_x,
                                     ew_net_type=c['ew_net_type'], out_fc=c['x2h_out_fc'])

    @classmethod
    def from_trace(cls, sd, cfg, trace, dtype=torch.float64):
        """The graph of block 0 of a `restate.forward(..., trace=trace)` run; a float64 gate is recomputed from the trace's x0."""
        e_w = trace['e_w'] if dtype == torch.float32 else None
        return cls(sd, cfg, trace['edge_index'], trace['edge_type'], trace['mask_ligand'], x0=trace['all_x'][0], e_w=e_w, dtype=dtype)


def row_error(got, want, inp, rows=None):
    """Per-row error of one layer's output:  |got - want|_inf / max(|want - inp|_inf, 0.01 * median_r |want - inp|_inf),
    i.e. relative to the size of the row's update, with a floor for rows the layer barely moves.  `rows`: boolean row selection."""
    got, want, inp = got.double(), want.double(), inp.double()
    if rows is not None:
        got, want, inp = got[rows], want[rows], inp[rows]
    upd = (want - inp).abs().amax(1)
    floor = 0.01 * upd.median()
    return (got - want).abs().amax(1) / torch.clamp(upd, min=float(floor))


def summary(err):
    """(max, 99.9th percentile) of a per-row error vector."""
    e = err.numpy()
    return float(e.max()), float(np.percentile(e, 99.9))
