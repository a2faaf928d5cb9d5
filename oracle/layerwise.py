"""One attention layer at a time, at any floating-point precision (TEST INFRASTRUCTURE, CPU only).

`restate.forward` chains all layers in fp32, so comparing the engine with it measures the rounding of the whole network at once.
The helpers here evaluate `restate.att_layer` on a given layer input -- typically the engine's own output of the previous layer --
in float64, so a comparison measures the rounding of that one layer only.  The graph, its edge types and the global edge gate are
the ones of the fp32 oracle's trace (the engine's `edge_index` is asserted bit-exact against it elsewhere).

`restate` builds its scatter buffers with `torch.zeros(...)`, so the float64 evaluation runs under `torch.set_default_dtype`;
`default_dtype` restores the previous default in every case.

`engine_layer_parity` runs that comparison against the engine for every layer of a network; it is shared by
tests/test_gpu_layer_parity.py and tests/test_gpu_workload_shapes.py, with the limits `LAYER_TOL`.
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


def embedding(sd, cfg, b, time_step=None, dtype=torch.float64):
    """The composed node features before block 0 (`restate.embed` then `compose_context`) of batch `b`, in `dtype`: protein rows
    W_p f + b_p with indicator 0, ligand rows W_l[:, v] + b_l (+ w_time t / T) with indicator 1.  Returns (h [N,128], mask_ligand)."""
    sdd = _cast({k: v for k, v in sd.items() if k.endswith('_atom_emb.weight') or k.endswith('_atom_emb.bias') or
                 k in ('betas', 'v_inference.2.weight')}, dtype)
    with default_dtype(dtype):
        h_p, h_l = restate.embed(sdd, cfg, b['protein_v'], b['init_ligand_v'], b['batch_ligand'], time_step)
        h, _, _, mask = restate.compose_context(h_p, h_l, b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    return h, mask


def head(sd, lig_h, dtype=torch.float64):
    """The atom-type head (`restate.head`: Linear, softplus with the threshold-20 branch, minus the fp32 ln 2, Linear) on `lig_h`."""
    sdd = _cast({k: v for k, v in sd.items() if k.startswith('v_inference.')}, dtype)
    with default_dtype(dtype):
        return restate.head(sdd, lig_h.to(dtype))


def block(sd, cfg, h, x, mask_ligand, batch_all, dtype=torch.float64):
    """One block of `restate.refine_net` from its input (h, x) [N,...] in the composed node order: the graph rebuilt from `x` as it
    is (fp32 coordinates; `restate.connect_edge`: `knn_graph_canonical` or `hybrid_graph_canonical`), the edge types, the global
    gate in `dtype` (`global_edge_weight`), then the block's num_layers attention layers in `dtype`.  Returns (h, x, edge_index, e_w)."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    edge_index = restate.connect_edge(x.float(), c, mask_ligand, batch_all)
    edge_type = restate.build_edge_type(edge_index, mask_ligand).argmax(-1)
    ref = LayerRef(sd, c, edge_index, edge_type, mask_ligand, x0=x, dtype=dtype)
    for l in range(c['num_layers']):
        h, x = ref(l, h, x)
    return h, x, edge_index, ref.e_w


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


# Largest per-row error (h, x) of one layer against float64 allowed per edge-MLP mode, about 3-4x the maximum measured on one
# NVIDIA H100 80GB HBM3 at a 400 W power limit (the kernels are deterministic).  The fp32 oracle's own error on the same inputs is
# 3e-7 - 9e-7 in h and up to 1.8e-4 in x.  Measured maxima, and the cases they cover:
#   every mode, k = 8, 32, 48 (test_layer_parity_every_mode):  tc3 h 8.7e-6 x 1.4e-4 | tc3v2 h 8.1e-6 x 8.6e-5 |
#                                                               tc6 h 2.5e-6 x 3.1e-5 | simt  h 5.7e-7 x 2.4e-5
#   tc3 (default), every other case of test_gpu_layer_parity.py, k >= 2:  h 1.22e-5 (x2h_out_fc)  x 8.9e-4 (the 40-graph batch, 1600 ligand rows)
#   tc3, k = 1:                                                h 1.27e-5                 x 1.53e-3
# The bf16-split modes keep ~16 mantissa bits per operand, hence ~1e-5 in h.  x is relative to the layer's displacement, a mean
# over 16 heads of signed terms (at k = 1, of one edge's terms only): rows where they nearly cancel amplify every mode's error, the
# fp32 oracle's too.  The k = 1 maximum gets its own x limit so that it does not loosen the check at every other k.
LAYER_TOL = {'tc3': (4e-5, 3e-3), 'tc3v2': (3e-5, 3e-4), 'tc6': (1e-5, 1e-4), 'simt': (2e-6, 8e-5)}
X_TOL_K1 = 5e-3                                        # tc3, k = 1


def _sorted_edges(ei):
    key = ei[1] * (int(ei.max()) + 1 if ei.numel() else 1) + ei[0]
    return ei[:, torch.argsort(key)]


def engine_layer_parity(label, cfg, sd, b, n_layers, make_model, dev, time_step=None, tag=''):
    """The engine cut after l = 1 .. n_layers layers against `LayerRef` in float64 on the engine's own output of l - 1 layers, on the
    fp32 oracle's graph of batch `b` (centred on the pockets); the engine's edge set must equal the oracle's.  `make_model(cfg, sd)`
    returns the engine's ScorePosNet3D on `dev` for a (cut) config and state dict.  Returns one row per layer:
    (layer, h err max, h p99.9, x err max, x p99.9, the fp32 oracle's 4 values)."""
    cfg = dict(cfg or {})
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    restate.forward(sd, dict(cfg, num_layers=1), pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'],
                    trace=tr, time_step=time_step)
    ref64 = LayerRef.from_trace(sd, cfg, tr)
    ref32 = LayerRef.from_trace(sd, cfg, tr, dtype=torch.float32)
    lig = tr['mask_ligand']
    hybrid = cfg.get('cutoff_mode') == 'hybrid'
    args = (pp.to(dev), b['protein_v'].to(dev), b['batch_protein'].to(dev), lp.to(dev), b['init_ligand_v'].to(dev), b['batch_ligand'].to(dev))
    kw = {} if time_step is None else {'time_step': time_step.to(dev)}
    h, x = tr['all_h'][0], tr['all_x'][0]
    rows = []
    for l in range(1, n_layers + 1):
        model = make_model(dict(cfg, num_layers=l), prefix_state_dict(sd, l))
        out = model(*args, **kw)
        ei = out['edge_index'].cpu()
        if hybrid:              # the engine's slot list is destination-sorted; the edge set must agree bit for bit
            assert torch.equal(_sorted_edges(ei), _sorted_edges(tr['edge_index']))
        else:
            assert torch.equal(ei, tr['edge_index'])
        h_gpu = out['final_h'].cpu()
        x_gpu = x.clone()
        x_gpu[lig] = out['pred_ligand_pos'].cpu()
        h64, x64 = ref64(l - 1, h, x)
        h32, x32 = ref32(l - 1, h, x)
        r = (l,) + summary(row_error(h_gpu, h64, h)) + summary(row_error(x_gpu, x64, x, lig)) + \
            summary(row_error(h32, h64, h)) + summary(row_error(x32, x64, x, lig))
        rows.append(r)
        print('%-28s %-6s layer %d  h %.2e / %.2e  x %.2e / %.2e   fp32 oracle: h %.2e / %.2e  x %.2e / %.2e' % ((label, tag) + r))
        h, x = h_gpu, x_gpu
        del model
    return rows


def check_layers(rows, mode='tc3', k=32):
    th, tx = LAYER_TOL[mode]
    if k == 1:
        tx = X_TOL_K1
    for r in rows:
        assert r[1] <= th and r[3] <= tx, 'layer %d: h %.3e (limit %.1e), x %.3e (limit %.1e)' % (r[0], r[1], th, r[3], tx)
