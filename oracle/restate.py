"""CPU restatement of targetdiff's denoising-sampling hot path (TEST INFRASTRUCTURE, see oracle/__init__.py).

Plain torch-CPU fp32, op by op, working directly on a reference-layout `state_dict` (SURVEY.md
Appendix D).  Every function cites the reference lines it restates (paths relative to the reference checkout).
Randomness never comes from an RNG here: the sampler consumes a *noise tape* (oracle.synth.make_tape)
in the reference's draw order.

Pinned against the reference itself (run under oracle/shims in the build container):
tests/test_oracle_vs_reference.py (bit-exact) and the committed vectors in tests/golden/.
Third-party arithmetic (torch_cluster knn, torch_scatter reduction order) is not in the reference
tree -> "parity unpinned" there; canonical semantics per SURVEY.md Appendix A.3/A.4.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .synth import DEFAULT_MODEL_CONFIG, GAUSSIAN_OFFSETS


# ----------------------------------------------------------------------------------------------
# a14  schedules                                   models/molopt_score_model.py:48-97,169-170,221-267
# ----------------------------------------------------------------------------------------------
def _sigmoid_betas(beta_start, beta_end, T):
    # models/molopt_score_model.py:72-74
    b = np.linspace(-6, 6, T)
    b = 1 / (np.exp(-b) + 1)
    return b * (beta_end - beta_start) + beta_start


def _cosine_alphas(T, s):
    # models/molopt_score_model.py:80-97 (returns sqrt of the per-step alpha ratio, clipped)
    steps = T + 1
    x = np.linspace(0, steps, steps)
    ac = np.cos(((x / steps) + s) / (1 + s) * np.pi * 0.5) ** 2
    ac = ac / ac[0]
    alphas = ac[1:] / ac[:-1]
    alphas = np.clip(alphas, a_min=0.001, a_max=1.)
    return np.sqrt(alphas)


def make_schedules(cfg=None):
    """The 15 fp32 tables of ScorePosNet3D.__init__ (models/molopt_score_model.py:221-267).
    fp64 numpy -> `.float()` exactly as `to_torch_const` (:104-107)."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    T = cfg['num_diffusion_timesteps']
    assert cfg['beta_schedule'] == 'sigmoid' and cfg['v_beta_schedule'] == 'cosine'
    betas = _sigmoid_betas(cfg['beta_start'], cfg['beta_end'], T)
    alphas = 1. - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1., ac[:-1])
    f = lambda a: torch.from_numpy(np.asarray(a)).float()
    out = {
        'betas': f(betas), 'alphas_cumprod': f(ac), 'alphas_cumprod_prev': f(ac_prev),
        'sqrt_alphas_cumprod': f(np.sqrt(ac)), 'sqrt_one_minus_alphas_cumprod': f(np.sqrt(1. - ac)),
        'sqrt_recip_alphas_cumprod': f(np.sqrt(1. / ac)), 'sqrt_recipm1_alphas_cumprod': f(np.sqrt(1. / ac - 1)),
        'posterior_mean_c0_coef': f(betas * np.sqrt(ac_prev) / (1. - ac)),
        'posterior_mean_ct_coef': f((1. - ac_prev) * np.sqrt(alphas) / (1. - ac)),
    }
    post_var = f(betas * (1. - ac_prev) / (1. - ac))
    out['posterior_var'] = post_var
    # :254 -- note: built from the *fp32* tensor, index 0 replaced by index 1, log taken in fp32->fp64 numpy
    out['posterior_logvar'] = f(np.log(np.append(post_var[1], post_var[1:])))
    alphas_v = _cosine_alphas(T, cfg['v_beta_s'])
    la = np.log(alphas_v)
    lca = np.cumsum(la)
    l1m = lambda a: np.log(1 - np.exp(a) + 1e-40)          # :169-170
    out['log_alphas_v'] = f(la)
    out['log_one_minus_alphas_v'] = f(l1m(la))
    out['log_alphas_cumprod_v'] = f(lca)
    out['log_one_minus_alphas_cumprod_v'] = f(l1m(lca))
    return out


# ----------------------------------------------------------------------------------------------
# a13  categorical / posterior helpers             models/molopt_score_model.py:124-175,371-428,706-708
# ----------------------------------------------------------------------------------------------
def extract(coef, t, batch):
    return coef[t][batch].unsqueeze(-1)                                    # :706-708


def index_to_log_onehot(x, num_classes):
    return torch.log(F.one_hot(x, num_classes).float().clamp(min=1e-30))   # :124-130


def log_add_exp(a, b):
    m = torch.max(a, b)                                                    # :173-175
    return m + torch.log(torch.exp(a - m) + torch.exp(b - m))


def q_v_pred_one_timestep(sd, log_vt_1, t, batch, K):
    la = extract(sd['log_alphas_v'], t, batch)                             # :371-381
    l1 = extract(sd['log_one_minus_alphas_v'], t, batch)
    return log_add_exp(log_vt_1 + la, l1 - np.log(K))


def q_v_pred(sd, log_v0, t, batch, K):
    la = extract(sd['log_alphas_cumprod_v'], t, batch)                     # :383-392
    l1 = extract(sd['log_one_minus_alphas_cumprod_v'], t, batch)
    return log_add_exp(log_v0 + la, l1 - np.log(K))


def q_v_posterior(sd, log_v0, log_vt, t, batch, K):
    tm1 = t - 1                                                            # :401-409
    tm1 = torch.where(tm1 < 0, torch.zeros_like(tm1), tm1)
    un = q_v_pred(sd, log_v0, tm1, batch, K) + q_v_pred_one_timestep(sd, log_vt, t, batch, K)
    return un - torch.logsumexp(un, dim=-1, keepdim=True)


def q_pos_posterior(sd, x0, xt, t, batch):
    return extract(sd['posterior_mean_c0_coef'], t, batch) * x0 + \
        extract(sd['posterior_mean_ct_coef'], t, batch) * xt               # :424-428


def log_sample_categorical_from_uniform(logits, uniform):
    g = -torch.log(-torch.log(uniform + 1e-30) + 1e-30)                    # :160-166
    return (g + logits).argmax(dim=-1)


def center_pos(protein_pos, ligand_pos, batch_protein, batch_ligand, mode='protein'):
    """models/molopt_score_model.py:110-120; scatter_mean = sequential sum / count."""
    if mode == 'none':
        return protein_pos, ligand_pos, 0.
    assert mode == 'protein'
    B = int(batch_protein.max()) + 1
    s = torch.zeros(B, 3).index_add_(0, batch_protein, protein_pos)
    cnt = torch.zeros(B).index_add_(0, batch_protein, torch.ones(len(batch_protein)))
    cnt[cnt < 1] = 1
    offset = s / cnt[:, None]
    return protein_pos - offset[batch_protein], ligand_pos - offset[batch_ligand], offset


# ----------------------------------------------------------------------------------------------
# a8/a9  shared NN bits                                            models/common.py:7-26,60-90,156-162
# ----------------------------------------------------------------------------------------------
def gaussian_smearing(dist, offset):
    coeff = -0.5 / (offset[1] - offset[0]).item() ** 2                     # common.py:17
    d = dist.view(-1, 1) - offset.view(1, -1)                              # common.py:25
    return torch.exp(coeff * torch.pow(d, 2))                              # common.py:26


def outer_product_type_gauss(edge_type_onehot, g):
    # common.py:83-90 for two vectors: out[e, t*20+j] = type[e,t]*g[e,j]  (int64 * f32 -> f32)
    out = edge_type_onehot.unsqueeze(-1) * g.unsqueeze(1)
    return out.view(out.shape[0], -1)


def mlp(sd, prefix, x):
    """Linear -> LayerNorm(eps=1e-5) -> ReLU -> Linear (common.py:60-80, norm=True, act_fn='relu')."""
    y = F.linear(x, sd[prefix + '.net.0.weight'], sd[prefix + '.net.0.bias'])
    y = F.layer_norm(y, (y.shape[-1],), sd[prefix + '.net.1.weight'], sd[prefix + '.net.1.bias'], 1e-5)
    y = F.relu(y)
    return F.linear(y, sd[prefix + '.net.3.weight'], sd[prefix + '.net.3.bias'])


# ----------------------------------------------------------------------------------------------
# a7  graph construction                                          models/uni_transformer.py:276-299
# ----------------------------------------------------------------------------------------------
def knn_graph_canonical(x, k, batch):
    """Canonical k-NN (SURVEY.md Appendix A.3): numpy, per graph, key = (fp32 d2, index) lexicographic.
    d2 = ((dx*dx)+(dy*dy))+(dz*dz) with every op rounded to fp32.  Returns int64 [2,E] (row0 src, row1 dst)."""
    xn = x.detach().cpu().numpy().astype(np.float32)
    bn = batch.detach().cpu().numpy()
    n = xn.shape[0]
    src_all, dst_all = [], []
    starts = np.flatnonzero(np.r_[True, bn[1:] != bn[:-1]]) if n else np.zeros(0, int)
    ends = np.r_[starts[1:], n]
    for s, e in zip(starts, ends):
        xg = xn[s:e]
        ng = e - s
        dx = xg[:, None, 0] - xg[None, :, 0]
        dy = xg[:, None, 1] - xg[None, :, 1]
        dz = xg[:, None, 2] - xg[None, :, 2]
        d2 = ((dx * dx).astype(np.float32) + (dy * dy).astype(np.float32)).astype(np.float32)
        d2 = (d2 + (dz * dz).astype(np.float32)).astype(np.float32)
        kk = min(k + 1, ng)
        idx = np.arange(ng)
        for i in range(ng):
            order = np.lexsort((idx, d2[i]))[:kk]       # primary d2, secondary index
            order = order[order != i]
            src_all.append(order + s)
            dst_all.append(np.full(len(order), i + s))
    src = np.concatenate(src_all) if src_all else np.zeros(0, np.int64)
    dst = np.concatenate(dst_all) if dst_all else np.zeros(0, np.int64)
    return torch.from_numpy(np.stack([src, dst]).astype(np.int64))


def hybrid_graph(x, k, mask_ligand, batch):
    """cutoff_mode='hybrid' (models/uni_transformer.py:281-283 -> models/common.py:165-212, add_p_index=True).  Per graph, in this
    edge order: ligand-ligand fully connected (dst-major, :167-171), for every ligand atom its k nearest PROTEIN atoms by
    torch.norm distance / torch.topk (:174-182), and for protein destinations the ordinary k-NN over all atoms of the graph
    (:196-203; nodes of a graph are protein atoms then ligand atoms after compose_context, so `all_index` is the identity)."""
    B = int(batch.max().item()) + 1 if len(batch) else 0
    out = []
    for g in range(B):
        lig = ((batch == g) & (mask_ligand == 1)).nonzero()[:, 0]                       # :190
        pro = ((batch == g) & (mask_ligand == 0)).nonzero()[:, 0]                       # :191
        dst = torch.repeat_interleave(lig, len(lig))                                    # :167
        src = lig.repeat(len(lig))                                                      # :168
        keep = dst != src
        ll = torch.stack([src[keep], dst[keep]])
        d = torch.norm(x[lig].unsqueeze(1) - x[pro].unsqueeze(0), p=2, dim=-1)         # :174-175
        nn_p = pro[torch.topk(d, k=k, largest=False, dim=1).indices]                    # :176-177
        pl = torch.stack([nn_p, lig.unsqueeze(1).repeat(1, k)], 0).view(2, -1)         # :178-182
        nodes = torch.cat([pro, lig])
        pe = knn_graph_canonical(x[nodes], k, torch.zeros(len(nodes), dtype=torch.long))   # :197
        pe = pe[:, pe[1] < len(pro)]                                                    # :198
        pe = torch.stack([nodes[pe[0]], nodes[pe[1]]], 0)                               # :199-202
        out.append(torch.cat([ll, pl, pe], -1))                                         # :205-206
    return torch.cat(out, -1) if out else torch.zeros(2, 0, dtype=torch.long)


def connect_edge(x, cfg, mask_ligand, batch):
    """_connect_edge (models/uni_transformer.py:276-286); 'radius' is a dead path in the reference (undefined self.r)."""
    if cfg['cutoff_mode'] == 'hybrid':
        return hybrid_graph(x, cfg['knn'], mask_ligand, batch)
    return knn_graph_canonical(x, cfg['knn'], batch)


def build_edge_type(edge_index, mask_ligand):
    """uni_transformer.py:288-299: L->L 0, L(src)->P(dst) 1, P(src)->L(dst) 2, P->P 3; one-hot int64 [E,4]."""
    src, dst = edge_index
    ns, nd = mask_ligand[src] == 1, mask_ligand[dst] == 1
    code = torch.zeros(len(src), dtype=torch.long)
    code[ns & nd] = 0
    code[ns & ~nd] = 1
    code[~ns & nd] = 2
    code[~ns & ~nd] = 3
    return F.one_hot(code, num_classes=4)


# ----------------------------------------------------------------------------------------------
# scatter ops in the reference's (CPU, sequential edge-order) semantics
# ----------------------------------------------------------------------------------------------
def scatter_softmax_rows(src, index, n):
    """torch_scatter.composite.scatter_softmax over dim 0 (call sites uni_transformer.py:73,135)."""
    idx = index[:, None].expand_as(src)
    mx = torch.zeros(n, src.shape[1]).scatter_reduce(0, idx, src, reduce='amax', include_self=False)
    ex = (src - mx.gather(0, idx)).exp_()
    sm = torch.zeros(n, src.shape[1]).scatter_add_(0, idx, ex)
    return ex.div(sm.gather(0, idx))


def scatter_sum_rows(src, index, n):
    """torch_scatter.scatter_sum over dim 0 (uni_transformer.py:78,139): scatter_add_ in edge order."""
    idx = index.view(-1, *([1] * (src.dim() - 1))).expand_as(src)
    return torch.zeros(n, *src.shape[1:]).scatter_add_(0, idx, src)


# ----------------------------------------------------------------------------------------------
# a10-a12  attention layers                                       models/uni_transformer.py:42-84,108-140,181-210
# ----------------------------------------------------------------------------------------------
def _edge_weight(sd, prefix, ew_net_type, r_feat, v, e_w):
    """The per-edge gate of one attention sub-layer (uni_transformer.py:58-66 / :121-129)."""
    if ew_net_type == 'r':
        return torch.sigmoid(F.linear(r_feat, sd[prefix + '.ew_net.0.weight'], sd[prefix + '.ew_net.0.bias']))     # :58-59,121-122
    if ew_net_type == 'm':
        if v is None:
            return 1.                                                                                           # h2x: :123-124
        H = sd[prefix + '.ew_net.0.weight'].shape[1]
        return torch.sigmoid(F.linear(v[..., :H], sd[prefix + '.ew_net.0.weight'], sd[prefix + '.ew_net.0.bias']))  # :60-61
    if e_w is not None:
        return e_w.view(-1, 1)                                                                                  # :62-63
    return 1.                                                                                                   # :64-65


def x2h_layer(sd, prefix, h, r_feat, edge_feat, edge_index, e_w, n_heads, ew_net_type='global', out_fc=False):
    N = h.size(0)
    src, dst = edge_index
    kv_input = torch.cat([edge_feat, torch.cat([r_feat, h[dst], h[src]], -1)], -1)       # :45-51
    H = h.shape[1]
    k = mlp(sd, prefix + '.hk_func', kv_input).view(-1, n_heads, H // n_heads)           # :54
    v = mlp(sd, prefix + '.hv_func', kv_input)                                           # :56
    v = v * _edge_weight(sd, prefix, ew_net_type, r_feat, v, e_w)                        # :58-66
    v = v.view(-1, n_heads, H // n_heads)
    q = mlp(sd, prefix + '.hq_func', h).view(-1, n_heads, H // n_heads)                  # :70
    alpha = scatter_softmax_rows((q[dst] * k / np.sqrt(k.shape[-1])).sum(-1), dst, N)    # :73-74
    m = alpha.unsqueeze(-1) * v                                                          # :77
    out = scatter_sum_rows(m, dst, N).view(-1, H)                                        # :78-79
    if out_fc:
        out = mlp(sd, prefix + '.node_output', torch.cat([out, h], -1))                  # :80-81
    return out + h                                                                       # :83


def h2x_layer(sd, prefix, h, rel_x, r_feat, edge_feat, edge_index, e_w, n_heads, ew_net_type='global'):
    N = h.size(0)
    src, dst = edge_index
    kv_input = torch.cat([edge_feat, torch.cat([r_feat, h[dst], h[src]], -1)], -1)       # :111-117
    H = h.shape[1]
    k = mlp(sd, prefix + '.xk_func', kv_input).view(-1, n_heads, H // n_heads)           # :119
    v = mlp(sd, prefix + '.xv_func', kv_input)                                           # :120
    v = v * _edge_weight(sd, prefix, ew_net_type, r_feat, None, e_w)                     # :121-129
    v = v.unsqueeze(-1) * rel_x.unsqueeze(1)                                             # :131
    q = mlp(sd, prefix + '.xq_func', h).view(-1, n_heads, H // n_heads)                  # :132
    alpha = scatter_softmax_rows((q[dst] * k / np.sqrt(k.shape[-1])).sum(-1), dst, N)    # :135
    m = alpha.unsqueeze(-1) * v                                                          # :138
    return scatter_sum_rows(m, dst, N).mean(1)                                           # :139-140


def att_layer(sd, prefix, h, x, edge_type, edge_index, mask_ligand, e_w, n_heads, fix_x=False, ew_net_type='global', out_fc=False):
    """AttentionLayerO2TwoUpdateNodeGeneral.forward, num_x2h=num_h2x=1, sync_twoup=False (:181-210)."""
    src, dst = edge_index
    offset = sd[prefix + '.distance_expansion.offset']
    rel_x = x[dst] - x[src]                                                              # :188
    dist = torch.norm(rel_x, p=2, dim=-1, keepdim=True)                                  # :189
    r_feat = outer_product_type_gauss(edge_type, gaussian_smearing(dist, offset))        # :194-195
    h_out = x2h_layer(sd, prefix + '.x2h_layers.0', h, r_feat, edge_type, edge_index, e_w, n_heads, ew_net_type, out_fc)
    r_feat = outer_product_type_gauss(edge_type, gaussian_smearing(dist, offset))        # :202-203
    dx = h2x_layer(sd, prefix + '.h2x_layers.0', h_out, rel_x, r_feat, edge_type, edge_index, e_w, n_heads, ew_net_type)
    if not fix_x:
        x = x + dx * mask_ligand[:, None]                                                # :205-206
    return h_out, x


def refine_net(sd, cfg, h, x, mask_ligand, batch, fix_x=False, edge_index=None, trace=None):
    """UniTransformerO2TwoUpdateGeneral.forward (uni_transformer.py:301-328): num_blocks x (k-NN graph, edge types, optional global
    gate, the SAME num_layers attention layers)."""
    assert cfg['cutoff_mode'] in ('knn', 'hybrid') and cfg['ew_net_type'] in ('global', 'r', 'm', 'none')
    given = edge_index
    for b in range(cfg['num_blocks']):                                                   # :306
        edge_index = given if (given is not None and b == 0) else connect_edge(x, cfg, mask_ligand, batch)   # :307
        src, dst = edge_index
        edge_type = build_edge_type(edge_index, mask_ligand)                             # :311
        e_w = None
        if cfg['ew_net_type'] == 'global':                                               # :312-318
            dist = torch.norm(x[dst] - x[src], p=2, dim=-1, keepdim=True)
            dist_feat = gaussian_smearing(dist, sd['refine_net.distance_expansion.offset'])
            e_w = torch.sigmoid(mlp(sd, 'refine_net.edge_pred_layer', dist_feat))
        if trace is not None and b == 0:
            trace.update(edge_index=edge_index, edge_type=edge_type.argmax(-1), e_w=None if e_w is None else e_w.view(-1), all_h=[h], all_x=[x])
        for l in range(cfg['num_layers']):
            h, x = att_layer(sd, 'refine_net.base_block.%d' % l, h, x, edge_type, edge_index, mask_ligand, e_w,
                             cfg['n_heads'], fix_x=fix_x, ew_net_type=cfg['ew_net_type'], out_fc=cfg['x2h_out_fc'])   # :320-321
            if trace is not None and b == 0:
                trace['all_h'].append(h)
                trace['all_x'].append(x)
        if trace is not None:
            trace.setdefault('block_edge_index', []).append(edge_index)
    return {'x': x, 'h': h}


# ----------------------------------------------------------------------------------------------
# a5/a6  forward                               models/molopt_score_model.py:313-368; models/common.py:120-137
# ----------------------------------------------------------------------------------------------
def compose_context(h_protein, h_ligand, pos_protein, pos_ligand, batch_protein, batch_ligand):
    batch_ctx = torch.cat([batch_protein, batch_ligand], dim=0)
    sort_idx = torch.sort(batch_ctx, stable=True).indices                                # common.py:126
    mask_ligand = torch.cat([torch.zeros(len(batch_protein)).bool(), torch.ones(len(batch_ligand)).bool()])[sort_idx]
    return (torch.cat([h_protein, h_ligand])[sort_idx], torch.cat([pos_protein, pos_ligand])[sort_idx],
            batch_ctx[sort_idx], mask_ligand)


def forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand,
            fix_x=False, trace=None, time_step=None):
    """ScorePosNet3D.forward, node_indicator=True (molopt_score_model.py:313-368); time_emb_dim = 0 or time_emb_mode 'simple'
    ('sin' cannot run in the reference: `time_feat` is [B, dim] but is concatenated with the [Nl, K] one-hot, :325-326)."""
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
    h_all, pos_all, batch_all, mask_ligand = compose_context(h_p, h_l, protein_pos, ligand_pos, batch_protein, batch_ligand)
    out = refine_net(sd, cfg, h_all, pos_all, mask_ligand, batch_all, fix_x=fix_x, trace=trace)   # :349
    final_pos, final_h = out['x'], out['h']
    lig_h = final_h[mask_ligand]                                                         # :350-351
    y = F.linear(lig_h, sd['v_inference.0.weight'], sd['v_inference.0.bias'])            # :307-311,352
    y = F.softplus(y) - torch.log(torch.tensor(2.0)).item()     # common.py:156-162 (shift = fp32 log 2)
    logits = F.linear(y, sd['v_inference.2.weight'], sd['v_inference.2.bias'])
    if trace is not None:
        trace.update(mask_ligand=mask_ligand, batch_all=batch_all)
    return {'pred_ligand_pos': final_pos[mask_ligand], 'pred_ligand_v': logits, 'final_h': final_h,
            'final_ligand_h': lig_h}


# ----------------------------------------------------------------------------------------------
# a4  the sampling loop                                        models/molopt_score_model.py:633-703
# ----------------------------------------------------------------------------------------------
def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand,
                     pos_noise, v_uniform, num_steps=None, center_pos_mode='protein', step_callback=None, pos_only=False):
    """Sampler (model_mean_type C0 or noise) driven by a noise tape: pos_noise [S,Nl,3], v_uniform [S,Nl,K].
    Returns the reference's dict ('pos','v','pos_traj','v_traj','v0_traj','vt_traj'), trajectories as lists."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    assert cfg['model_mean_type'] in ('C0', 'noise')
    T = sd['betas'].shape[0]
    K = sd['v_inference.2.weight'].shape[0]
    if num_steps is None:
        num_steps = T
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, ligand_pos, offset = center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        # mode 'none' returns the float 0. (:118-119) and the reference's own `offset[batch_ligand]` (:691,695) then raises TypeError;
        # the engine defines the obvious meaning (no shift), restated here so that the extension can be checked
        offset = torch.zeros(num_graphs, 3)
    ligand_v = init_ligand_v
    pos_traj, v_traj, v0_traj, vt_traj = [], [], [], []
    time_seq = list(reversed(range(T - num_steps, T)))                                   # :649
    for s, i in enumerate(time_seq):
        t = torch.full((num_graphs,), i, dtype=torch.long)                               # :651
        preds = forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step=t)
        pos0, v0 = preds['pred_ligand_pos'], preds['pred_ligand_v']                      # :667-669
        if cfg['model_mean_type'] == 'noise':                                            # :663-666 with :419-422
            eps = pos0 - ligand_pos
            pos0 = extract(sd['sqrt_recip_alphas_cumprod'], t, batch_ligand) * ligand_pos - \
                extract(sd['sqrt_recipm1_alphas_cumprod'], t, batch_ligand) * eps
        pos_mean = q_pos_posterior(sd, pos0, ligand_pos, t, batch_ligand)                # :673
        logvar = extract(sd['posterior_logvar'], t, batch_ligand)                        # :674
        nonzero = (1 - (t == 0).float())[batch_ligand].unsqueeze(-1)                     # :676
        ligand_pos = pos_mean + nonzero * (0.5 * logvar).exp() * pos_noise[s]            # :677-679
        if not pos_only:                                                                 # :681
            log_v_recon = F.log_softmax(v0, dim=-1)                                      # :682
            log_v = index_to_log_onehot(ligand_v, K)                                     # :683
            log_model_prob = q_v_posterior(sd, log_v_recon, log_v, t, batch_ligand, K)   # :684
            ligand_v = log_sample_categorical_from_uniform(log_model_prob, v_uniform[s])  # :685
            v0_traj.append(log_v_recon.clone()); vt_traj.append(log_model_prob.clone())  # :687-688
        pos_traj.append((ligand_pos + offset[batch_ligand]).clone())                     # :691-692
        v_traj.append(ligand_v.clone())                                                  # :693
        if step_callback is not None:
            step_callback(s, i, preds, ligand_pos, ligand_v)
    return {'pos': ligand_pos + offset[batch_ligand], 'v': ligand_v, 'pos_traj': pos_traj, 'v_traj': v_traj,
            'v0_traj': v0_traj, 'vt_traj': vt_traj}


# ----------------------------------------------------------------------------------------------
# a1/a2  the sampling driver and the ligand-size prior    scripts/sample_diffusion.py:31-116; utils/evaluation/atom_num.py:9-26
# ----------------------------------------------------------------------------------------------
def get_space_size(pocket_3d_pos):
    """utils/evaluation/atom_num.py:9-12: median of the 10 largest pairwise distances (scipy pdist, fp64)."""
    from scipy import spatial as sc_spatial
    d = sc_spatial.distance.pdist(pocket_3d_pos, metric='euclidean')
    return np.median(np.sort(d)[::-1][:10])


def sample_atom_num(space_size, prior):
    """utils/evaluation/atom_num.py:15-26 on the empirical table `prior` = {'bounds': [...], 'bins': [{'num_atoms', 'prob'}, ...]}
    (utils/evaluation/atom_num_config.py, a constant table); numpy's GLOBAL RNG like the reference."""
    idx = len(prior['bounds'])
    for i, b in enumerate(prior['bounds']):
        if b > space_size:
            idx = i
            break
    b = prior['bins'][idx]
    return np.random.choice(b['num_atoms'], p=b['prob'])


def sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, batch_size=16, num_steps=None,
                            pos_only=False, center_pos_mode='protein', sample_num_atoms='prior', ligand_v_full=None):
    """scripts/sample_diffusion.py:31-116 on CPU.  Randomness comes from numpy's / torch's GLOBAL CPU generators in the reference's
    order (seed them like utils/misc.py:58-61): per batch the size draws (:49), randn_like(center) (:63), rand_like(uniform logits)
    (:69 -> models/molopt_score_model.py:161), then per step randn_like(pos) / rand_like(log prob) (models/molopt_score_model.py:678,685),
    which are pre-drawn here in that interleaved order and handed to `sample_diffusion` as a tape.
    Returns the reference's 7-tuple (positions float64 numpy, trajectories [steps, atoms, ...]); the time list holds zeros."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['ligand_atom_emb.weight'].shape[1]
    T = sd['betas'].shape[0]
    S = T if num_steps is None else num_steps
    all_pos, all_v, all_pos_traj, all_v_traj, all_v0_traj, all_vt_traj, time_list = [], [], [], [], [], [], []
    num_batch = int(np.ceil(num_samples / batch_size))                                   # :38
    current_i = 0
    n_prot = protein_pos.shape[0]
    for i in range(num_batch):
        n_data = batch_size if i < num_batch - 1 else num_samples - batch_size * (num_batch - 1)    # :41
        batch_protein = torch.repeat_interleave(torch.arange(n_data), n_prot)            # Batch.from_data_list of n_data clones, :42
        ppos = protein_pos.repeat(n_data, 1)
        pfeat = protein_atom_feature.float().repeat(n_data, 1)
        if sample_num_atoms == 'prior':                                                  # :47-50
            pocket_size = get_space_size(protein_pos.detach().cpu().numpy())
            sizes = [int(sample_atom_num(pocket_size, prior)) for _ in range(n_data)]
        elif sample_num_atoms == 'range':                                                # :51-53
            sizes = list(range(current_i + 1, current_i + n_data + 1))
        else:
            raise ValueError(sample_num_atoms)
        batch_ligand = torch.repeat_interleave(torch.arange(n_data), torch.tensor(sizes))
        s3 = torch.zeros(n_data, 3).index_add_(0, batch_protein, ppos)                   # scatter_mean, :61
        center = s3 / torch.zeros(n_data).index_add_(0, batch_protein, torch.ones(len(batch_protein)))[:, None]
        bc = center[batch_ligand]
        init_pos = bc + torch.randn_like(bc)                                             # :63
        if pos_only:
            init_v = ligand_v_full.repeat(n_data)                                        # :67
        else:
            init_v = log_sample_categorical_from_uniform(torch.zeros(len(batch_ligand), K),
                                                         torch.rand(len(batch_ligand), K))   # :69-70
        pn = torch.empty(S, len(batch_ligand), 3)
        vu = torch.zeros(S, len(batch_ligand), K)
        for st in range(S):
            pn[st] = torch.randn(len(batch_ligand), 3)
            if not pos_only:
                vu[st] = torch.rand(len(batch_ligand), K)
        r = sample_diffusion(sd, c, ppos, pfeat, batch_protein, init_pos, init_v, batch_ligand, pn, vu, num_steps=num_steps,
                             center_pos_mode=center_pos_mode, pos_only=pos_only)         # :72-82
        cum = np.cumsum([0] + sizes)                                                     # :86
        pos = r['pos'].numpy().astype(np.float64)
        all_pos += [pos[cum[k]:cum[k + 1]] for k in range(n_data)]                       # :87-89
        ptraj = torch.stack(r['pos_traj']).numpy().astype(np.float64)
        all_pos_traj += [ptraj[:, cum[k]:cum[k + 1]] for k in range(n_data)]             # :91-98
        v = r['v'].numpy()
        all_v += [v[cum[k]:cum[k + 1]] for k in range(n_data)]                           # :101-102
        vtraj = torch.stack(r['v_traj']).numpy()
        all_v_traj += [vtraj[:, cum[k]:cum[k + 1]] for k in range(n_data)]               # :104-105
        if not pos_only:                                                                 # :107-111
            v0 = torch.stack(r['v0_traj']).numpy()
            vt = torch.stack(r['vt_traj']).numpy()
            all_v0_traj += [v0[:, cum[k]:cum[k + 1]] for k in range(n_data)]
            all_vt_traj += [vt[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        time_list.append(0.0)
        current_i += n_data
    return all_pos, all_v, all_pos_traj, all_v_traj, all_v0_traj, all_vt_traj, time_list


# ----------------------------------------------------------------------------------------------
# n3  likelihood estimation (second consumer of `forward`)     models/molopt_score_model.py:133-155,411-438,470-489,565-617
# ----------------------------------------------------------------------------------------------
def _normal_kl(mean1, logvar1, mean2, logvar2):
    d = mean1 - mean2                                                                    # :143-148
    return (0.5 * (-1.0 + logvar2 - logvar1 + torch.exp(logvar1 - logvar2) + d ** 2 * torch.exp(-logvar2))).sum(-1)


def _scatter_mean_rows(v, batch, B):
    s = torch.zeros(B, dtype=v.dtype).index_add_(0, batch, v)
    c = torch.zeros(B, dtype=v.dtype).index_add_(0, batch, torch.ones_like(v))
    c[c < 1] = 1
    return s / c


def likelihood_estimation(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step,
                          pos_noise=None, v_uniform=None):
    """ScorePosNet3D.likelihood_estimation (:565-617): per-graph (kl_pos, kl_v) at `time_step` [B] (< T), or the two prior KL
    terms when time_step == T everywhere.  RNG replaced by `pos_noise` [Nl,3] (the in-place normal_ of :581-582) and
    `v_uniform` [Nl,K] (rand_like inside q_v_sample, :394-398 via :160-166)."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    T = c['num_diffusion_timesteps']
    K = sd['ligand_atom_emb.weight'].shape[1]
    B = int(batch_protein.max()) + 1
    protein_pos, ligand_pos, _ = center_pos(protein_pos, ligand_pos, batch_protein, batch_ligand, 'protein')
    if bool((time_step == T).all()):
        last = torch.full((B,), T - 1, dtype=torch.long)
        a_pos = extract(sd['alphas_cumprod'], last, batch_ligand)                        # :430-438
        mean = a_pos.sqrt() * ligand_pos
        logvar = torch.log((1.0 - a_pos).sqrt())
        kl_pos = _scatter_mean_rows(_normal_kl(torch.zeros_like(mean), torch.zeros_like(logvar), mean, logvar), batch_ligand, B)
        # :573 passes batch_ligand (graph ids) where atom types are expected -- restated as written
        log_v0 = index_to_log_onehot(batch_ligand, K)
        log_qT = q_v_pred(sd, log_v0, last, batch_ligand, K)                             # :411-417
        log_half = -torch.log(K * torch.ones_like(log_qT))
        kl_v = _scatter_mean_rows((log_qT.exp() * (log_qT - log_half)).sum(1), batch_ligand, B)
        return kl_pos, kl_v
    assert bool((time_step < T).all())
    a_pos = sd['alphas_cumprod'].index_select(0, time_step)[batch_ligand].unsqueeze(-1)  # :578-579
    xt = a_pos.sqrt() * ligand_pos + (1.0 - a_pos).sqrt() * pos_noise                    # :583
    log_v0 = index_to_log_onehot(ligand_v, K)
    vt = log_sample_categorical_from_uniform(q_v_pred(sd, log_v0, time_step, batch_ligand, K), v_uniform)   # :586
    log_vt = index_to_log_onehot(vt, K)
    out = forward(sd, cfg, protein_pos, protein_v, batch_protein, xt, vt, batch_ligand)  # :588-597
    mean_model = q_pos_posterior(sd, out['pred_ligand_pos'], xt, time_step, batch_ligand)   # :600-603
    log_recon = F.log_softmax(out['pred_ligand_v'], dim=-1)
    log_model = q_v_posterior(sd, log_recon, log_vt, time_step, batch_ligand, K)
    log_true = q_v_posterior(sd, log_v0, log_vt, time_step, batch_ligand, K)
    mask = (time_step == 0).float()[batch_ligand]
    # position term (:470-482)
    logvar = extract(sd['posterior_logvar'], time_step, batch_ligand)
    mean_true = q_pos_posterior(sd, ligand_pos, xt, time_step, batch_ligand)
    kl_p = _normal_kl(mean_true, logvar, mean_model, logvar) / np.log(2.)
    ls = 0.5 * logvar
    nll_p = -((-((ligand_pos - mean_model) ** 2) / (2 * torch.exp(ls * 2)) - ls - np.log(np.sqrt(2 * np.pi))).sum(-1))
    kl_pos = _scatter_mean_rows(mask * nll_p + (1. - mask) * kl_p, batch_ligand, B)
    # type term (:484-489)
    kl_c = (log_true.exp() * (log_true - log_model)).sum(1)
    nll_c = -(log_v0.exp() * log_model).sum(1)
    kl_v = _scatter_mean_rows(mask * nll_c + (1. - mask) * kl_c, batch_ligand, B)
    return kl_pos, kl_v


# ----------------------------------------------------------------------------------------------
# n4  stability screen of generated molecules                      utils/evaluation/analyze.py:6-44,90-143
# ----------------------------------------------------------------------------------------------
_ELEMENTS = ['H', 'C', 'N', 'O', 'F', 'P', 'S', 'Cl']
_Z_TO_EL = {1: 0, 6: 1, 7: 2, 8: 3, 9: 4, 15: 5, 16: 6, 17: 7}                           # atom_encoder / atom_decoder, :6-7
_BONDS1 = [[74, 109, 101, 96, 92, 144, 134, 127], [109, 154, 147, 143, 135, 184, 182, 177], [101, 147, 145, 140, 136, 177, 168, 175],
           [96, 143, 140, 148, 142, 163, 151, 164], [92, 135, 136, 142, 142, 156, 158, 166], [144, 184, 177, 163, 156, 221, 210, 203],
           [134, 182, 168, 151, 158, 210, 204, 207], [127, 177, 175, 164, 166, 203, 207, 199]]                                       # :10-18
_BONDS2 = [[-1] * 8, [-1, 134, 129, 120, -1, -1, 160, -1], [-1, 129, 125, 121, -1, -1, -1, -1], [-1, 120, 121, 121, -1, 150, -1, -1],
           [-1] * 8, [-1, -1, -1, 150, -1, -1, 186, -1], [-1, 160, -1, -1, -1, 186, -1, -1], [-1] * 8]                              # :21-29
_BONDS3 = [[-1] * 8, [-1, 120, 116, 113, -1, -1, -1, -1], [-1, 116, 110, -1, -1, -1, -1, -1], [-1, 113, -1, -1, -1, -1, -1, -1],
           [-1] * 8, [-1] * 8, [-1] * 8, [-1] * 8]                                                                                   # :31-39
_ALLOWED = [1, 4, 3, 2, 1, 5, 4, 1]                                                                                                  # :44


def get_bond_order(e1, e2, distance):
    d = 100 * distance                                                                   # :91
    if d < _BONDS1[e1][e2] + 10:                                                         # margin1, :94
        if d < _BONDS2[e1][e2] + 5:                                                      # :95-96
            if d < _BONDS3[e1][e2] + 3:                                                  # :97-98
                return 3
            return 2
        return 1
    return 0


def check_stability(positions, atom_type, hs=False):
    """analyze.py:106-143 -> (molecule_stable, nr_stable_atoms, n_atoms, nr_bonds); positions float64 [n,3], atom_type atomic numbers."""
    positions = np.asarray(positions, dtype=np.float64)
    n = len(positions)
    nr_bonds = np.zeros(n, dtype='int')
    for i in range(n):
        for j in range(i + 1, n):
            dist = np.sqrt(np.sum((positions[i] - positions[j]) ** 2))                   # :117-119
            order = get_bond_order(_Z_TO_EL[int(atom_type[i])], _Z_TO_EL[int(atom_type[j])], dist)
            nr_bonds[i] += order
            nr_bonds[j] += order
    stable = 0
    for z, nb in zip(atom_type, nr_bonds):
        a = _ALLOWED[_Z_TO_EL[int(z)]]
        stable += int(a == nb) if hs else int(a >= nb > 0)                               # :130-133
    return stable == n, stable, n, nr_bonds
