"""CPU restatement of the layer forms of AttentionLayerO2TwoUpdateNodeGeneral (num_x2h, num_h2x, sync_twoup; reference
models/uni_transformer.py:143-210) and of forward(..., return_all=True) (models/molopt_score_model.py:360-367,
models/uni_transformer.py:303-327) (TEST INFRASTRUCTURE, see oracle/__init__.py).

`oracle.restate` restates the default form (one x2h and one h2x sub-layer per layer, sync_twoup = False).  This module builds the
general form from restate's own sub-layers, graph construction, embeddings, head and posterior helpers, so for the default form every
function here performs the same operations as its restate counterpart (tests/test_layer_forms.py checks bit-identity).  It is pinned
against the unmodified reference by tests/test_layer_forms.py (tests/golden/reference_pins_layer_forms.pt, oracle/make_layer_form_pins.py).
`LayerFormRef` and `engine_layer_parity` are the one-layer float64 counterparts of oracle.layerwise's for these forms.
"""
import torch
import torch.nn.functional as F

from . import layerwise, restate
from .synth import DEFAULT_MODEL_CONFIG


def form(cfg):
    """(num_x2h, num_h2x, sync_twoup) of a model config (reference defaults for absent keys)."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    return int(c['num_x2h']), int(c['num_h2x']), bool(c['sync_twoup'])


def att_layer(sd, prefix, h, x, edge_type, edge_index, mask_ligand, e_w, n_heads, fix_x=False, ew_net_type='global', out_fc=False,
              num_x2h=1, num_h2x=1, sync_twoup=False):
    """AttentionLayerO2TwoUpdateNodeGeneral.forward (:181-210): num_x2h feature updates in sequence on the layer's input coordinates,
    then num_h2x coordinate updates, each reading the x2h output (or, with sync_twoup, the layer's input h) and the edge lengths of
    the coordinates the previous one moved.  Returns the x2h output as h."""
    src, dst = edge_index
    offset = sd[prefix + '.distance_expansion.offset']
    rel_x = x[dst] - x[src]                                                              # :188
    dist = torch.norm(rel_x, p=2, dim=-1, keepdim=True)                                  # :189
    h_in = h
    for i in range(num_x2h):                                                             # :193-197
        r_feat = restate.outer_product_type_gauss(edge_type, restate.gaussian_smearing(dist, offset))       # :194-195
        h_in = restate.x2h_layer(sd, prefix + '.x2h_layers.%d' % i, h_in, r_feat, edge_type, edge_index, e_w, n_heads, ew_net_type, out_fc)
    h_out = h_in                                                                         # :198
    new_h = h if sync_twoup else h_out                                                   # :200
    for i in range(num_h2x):                                                             # :201-208
        r_feat = restate.outer_product_type_gauss(edge_type, restate.gaussian_smearing(dist, offset))       # :202-203
        dx = restate.h2x_layer(sd, prefix + '.h2x_layers.%d' % i, new_h, rel_x, r_feat, edge_type, edge_index, e_w, n_heads, ew_net_type)
        if not fix_x:
            x = x + dx * mask_ligand[:, None]                                            # :205-206
        rel_x = x[dst] - x[src]                                                          # :207
        dist = torch.norm(rel_x, p=2, dim=-1, keepdim=True)                              # :208
    return h_out, x


def refine_net(sd, cfg, h, x, mask_ligand, batch, fix_x=False, trace=None, return_all=False):
    """UniTransformerO2TwoUpdateGeneral.forward (uni_transformer.py:301-328) with the general layer form; `return_all`: also x and h
    before block 0 and after every block (:303-304,322-327).  `trace` as restate.refine_net."""
    assert cfg['cutoff_mode'] in ('knn', 'hybrid') and cfg['ew_net_type'] in ('global', 'r', 'm', 'none')
    nx, nh, sync = form(cfg)
    all_x, all_h = [x], [h]
    for b in range(cfg['num_blocks']):                                                   # :306
        edge_index = restate.connect_edge(x, cfg, mask_ligand, batch)                    # :307
        src, dst = edge_index
        edge_type = restate.build_edge_type(edge_index, mask_ligand)                     # :311
        e_w = None
        if cfg['ew_net_type'] == 'global':                                               # :312-318
            dist = torch.norm(x[dst] - x[src], p=2, dim=-1, keepdim=True)
            dist_feat = restate.gaussian_smearing(dist, sd['refine_net.distance_expansion.offset'])
            e_w = torch.sigmoid(restate.mlp(sd, 'refine_net.edge_pred_layer', dist_feat))
        if trace is not None and b == 0:
            trace.update(edge_index=edge_index, edge_type=edge_type.argmax(-1), e_w=None if e_w is None else e_w.view(-1), all_h=[h], all_x=[x])
        for l in range(cfg['num_layers']):
            h, x = att_layer(sd, 'refine_net.base_block.%d' % l, h, x, edge_type, edge_index, mask_ligand, e_w, cfg['n_heads'], fix_x=fix_x,
                             ew_net_type=cfg['ew_net_type'], out_fc=cfg['x2h_out_fc'], num_x2h=nx, num_h2x=nh, sync_twoup=sync)   # :320-321
            if trace is not None and b == 0:
                trace['all_h'].append(h)
                trace['all_x'].append(x)
        if trace is not None:
            trace.setdefault('block_edge_index', []).append(edge_index)
        all_x.append(x)                                                                  # :322-323
        all_h.append(h)
    out = {'x': x, 'h': h}
    if return_all:
        out.update(all_x=all_x, all_h=all_h)
    return out


def v_inference(sd, lig_h):
    """The type head (molopt_score_model.py:307-311,352), as in restate.forward."""
    y = F.linear(lig_h, sd['v_inference.0.weight'], sd['v_inference.0.bias'])
    y = F.softplus(y) - torch.log(torch.tensor(2.0)).item()     # common.py:156-162 (shift = fp32 log 2)
    return F.linear(y, sd['v_inference.2.weight'], sd['v_inference.2.bias'])


def forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, fix_x=False, trace=None, time_step=None,
            return_all=False):
    """restate.forward with the general layer form; `return_all` adds 'layer_pred_ligand_pos' / 'layer_pred_ligand_v', one entry
    before block 0 and one after every block (molopt_score_model.py:360-367)."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    assert cfg['node_indicator'] and (cfg['time_emb_dim'] == 0 or cfg['time_emb_mode'] == 'simple')
    T = sd['betas'].shape[0]
    K = sd['ligand_atom_emb.weight'].shape[1] - (1 if cfg['time_emb_dim'] > 0 else 0)
    lig_feat = F.one_hot(ligand_v, K).float()                                            # :317
    if cfg['time_emb_dim'] > 0:                                                          # :319-324
        lig_feat = torch.cat([lig_feat, (time_step / T)[batch_ligand].unsqueeze(-1)], -1)
    h_p = F.linear(protein_v, sd['protein_atom_emb.weight'], sd['protein_atom_emb.bias'])  # :333
    h_l = F.linear(lig_feat, sd['ligand_atom_emb.weight'], sd['ligand_atom_emb.bias'])     # :334
    h_p = torch.cat([h_p, torch.zeros(len(h_p), 1)], -1)                                 # :336-338
    h_l = torch.cat([h_l, torch.ones(len(h_l), 1)], -1)
    h_all, pos_all, batch_all, mask_ligand = restate.compose_context(h_p, h_l, protein_pos, ligand_pos, batch_protein, batch_ligand)
    out = refine_net(sd, cfg, h_all, pos_all, mask_ligand, batch_all, fix_x=fix_x, trace=trace, return_all=return_all)   # :349
    final_pos, final_h = out['x'], out['h']
    lig_h = final_h[mask_ligand]                                                         # :350-351
    if trace is not None:
        trace.update(mask_ligand=mask_ligand, batch_all=batch_all)
    preds = {'pred_ligand_pos': final_pos[mask_ligand], 'pred_ligand_v': v_inference(sd, lig_h), 'final_h': final_h, 'final_ligand_h': lig_h}
    if return_all:                                                                       # :360-367
        preds.update(layer_pred_ligand_pos=[p[mask_ligand] for p in out['all_x']],
                     layer_pred_ligand_v=[v_inference(sd, hh[mask_ligand]) for hh in out['all_h']])
    return preds


def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand, pos_noise, v_uniform,
                     num_steps=None, center_pos_mode='protein'):
    """restate.sample_diffusion (models/molopt_score_model.py:633-703, noise tape) with the general layer form."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    assert cfg['model_mean_type'] in ('C0', 'noise')
    T = sd['betas'].shape[0]
    K = sd['v_inference.2.weight'].shape[0]
    num_steps = T if num_steps is None else num_steps
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, ligand_pos, offset = restate.center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        offset = torch.zeros(num_graphs, 3)
    ligand_v = init_ligand_v
    pos_traj, v_traj, v0_traj, vt_traj = [], [], [], []
    for s, i in enumerate(reversed(range(T - num_steps, T))):                            # :649
        t = torch.full((num_graphs,), i, dtype=torch.long)                               # :651
        preds = forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step=t)
        pos0, v0 = preds['pred_ligand_pos'], preds['pred_ligand_v']                      # :667-669
        if cfg['model_mean_type'] == 'noise':                                            # :663-666 with :419-422
            eps = pos0 - ligand_pos
            pos0 = restate.extract(sd['sqrt_recip_alphas_cumprod'], t, batch_ligand) * ligand_pos - \
                restate.extract(sd['sqrt_recipm1_alphas_cumprod'], t, batch_ligand) * eps
        pos_mean = restate.q_pos_posterior(sd, pos0, ligand_pos, t, batch_ligand)        # :673
        logvar = restate.extract(sd['posterior_logvar'], t, batch_ligand)                # :674
        nonzero = (1 - (t == 0).float())[batch_ligand].unsqueeze(-1)                     # :676
        ligand_pos = pos_mean + nonzero * (0.5 * logvar).exp() * pos_noise[s]            # :677-679
        log_v_recon = F.log_softmax(v0, dim=-1)                                          # :682
        log_v = restate.index_to_log_onehot(ligand_v, K)                                 # :683
        log_model_prob = restate.q_v_posterior(sd, log_v_recon, log_v, t, batch_ligand, K)   # :684
        ligand_v = restate.log_sample_categorical_from_uniform(log_model_prob, v_uniform[s])  # :685
        v0_traj.append(log_v_recon.clone()); vt_traj.append(log_model_prob.clone())      # :687-688
        pos_traj.append((ligand_pos + offset[batch_ligand]).clone())                     # :691-692
        v_traj.append(ligand_v.clone())                                                  # :693
    return {'pos': ligand_pos + offset[batch_ligand], 'v': ligand_v, 'pos_traj': pos_traj, 'v_traj': v_traj,
            'v0_traj': v0_traj, 'vt_traj': vt_traj}


class LayerFormRef(layerwise.LayerRef):
    """oracle.layerwise.LayerRef for the general layer form of `cfg`: attention layer l at any floating-point precision."""

    def __call__(self, l, h, x, fix_x=False):
        c = self.cfg
        nx, nh, sync = form(c)
        with layerwise.default_dtype(self.dtype):
            return att_layer(self.sd, 'refine_net.base_block.%d' % l, h.to(self.dtype), x.to(self.dtype), self.edge_type, self.edge_index,
                             self.mask_ligand, self.e_w, c['n_heads'], fix_x=fix_x, ew_net_type=c['ew_net_type'], out_fc=c['x2h_out_fc'],
                             num_x2h=nx, num_h2x=nh, sync_twoup=sync)


def engine_layer_parity(label, cfg, sd, b, n_layers, make_model, dev):
    """oracle.layerwise.engine_layer_parity for the general layer form: the engine cut after l = 1 .. n_layers layers against
    LayerFormRef in float64 on the engine's own output of l - 1 layers, on the fp32 oracle's graph of batch `b` (block 0).  Returns one
    row per layer: (layer, h err max, h p99.9, x err max, x p99.9, the fp32 oracle's 4 values)."""
    cfg = dict(cfg or {})
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    forward(sd, dict(cfg, num_layers=1), pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    ref64 = LayerFormRef.from_trace(sd, cfg, tr)
    ref32 = LayerFormRef.from_trace(sd, cfg, tr, dtype=torch.float32)
    lig = tr['mask_ligand']
    hybrid = cfg.get('cutoff_mode') == 'hybrid'
    args = (pp.to(dev), b['protein_v'].to(dev), b['batch_protein'].to(dev), lp.to(dev), b['init_ligand_v'].to(dev), b['batch_ligand'].to(dev))
    h, x = tr['all_h'][0], tr['all_x'][0]
    rows = []
    for l in range(1, n_layers + 1):
        model = make_model(dict(cfg, num_layers=l), layerwise.prefix_state_dict(sd, l))
        out = model(*args)
        ei = out['edge_index'].cpu()
        if hybrid:
            assert torch.equal(layerwise._sorted_edges(ei), layerwise._sorted_edges(tr['edge_index']))
        else:
            assert torch.equal(ei, tr['edge_index'])
        h_gpu = out['final_h'].cpu()
        x_gpu = x.clone()
        x_gpu[lig] = out['pred_ligand_pos'].cpu()
        h64, x64 = ref64(l - 1, h, x)
        h32, x32 = ref32(l - 1, h, x)
        r = (l,) + layerwise.summary(layerwise.row_error(h_gpu, h64, h)) + layerwise.summary(layerwise.row_error(x_gpu, x64, x, lig)) + \
            layerwise.summary(layerwise.row_error(h32, h64, h)) + layerwise.summary(layerwise.row_error(x32, x64, x, lig))
        rows.append(r)
        print('%-28s layer %d  h %.2e / %.2e  x %.2e / %.2e   fp32 oracle: h %.2e / %.2e  x %.2e / %.2e' % ((label,) + r))
        h, x = h_gpu, x_gpu
        del model
    return rows
