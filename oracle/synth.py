"""Seeded synthetic inputs shared by tests/, smoke() and bench.py (test infrastructure).

Synthetic pocket recipe: SURVEY.md section 8(d).  Weights: a deterministic state_dict with the
reference's 384-entry layout (SURVEY.md Appendix D; reference models/molopt_score_model.py:236-311,
models/uni_transformer.py:241-274, models/common.py:63-77) drawn from a CPU torch.Generator, so the
same weights can be rebuilt anywhere, without the reference checkout.
"""
import math

import numpy as np
import torch

# reference configs/training.yml:9-42 (values only; the product has its own loader)
DEFAULT_MODEL_CONFIG = dict(
    model_mean_type='C0', beta_schedule='sigmoid', beta_start=1.e-7, beta_end=2.e-3,
    v_beta_schedule='cosine', v_beta_s=0.01, num_diffusion_timesteps=1000, loss_v_weight=100.,
    sample_time_method='symmetric', time_emb_dim=0, time_emb_mode='simple', center_pos_mode='protein',
    node_indicator=True, model_type='uni_o2', num_blocks=1, num_layers=9, hidden_dim=128, n_heads=16,
    edge_feat_dim=4, num_r_gaussian=20, knn=32, num_node_types=8, act_fn='relu', norm=True,
    cutoff_mode='knn', ew_net_type='global', num_x2h=1, num_h2x=1, r_max=10., x2h_out_fc=False,
    sync_twoup=False,
)

PROTEIN_FEATURE_DIM = 27   # reference utils/transforms.py:119-124 (6 elements + 20 AA + backbone flag)
LIGAND_NUM_CLASSES = 13    # reference utils/transforms.py:48-62 ('add_aromatic')

# reference models/common.py:15 (fixed_offset=True)
GAUSSIAN_OFFSETS = [0, 1, 1.25, 1.5, 1.75, 2, 2.25, 2.5, 2.75, 3, 3.5, 4, 4.5, 5, 5.5, 6, 7, 8, 9, 10]

SCHEDULE_KEYS = [
    'betas', 'alphas_cumprod', 'alphas_cumprod_prev', 'sqrt_alphas_cumprod', 'sqrt_one_minus_alphas_cumprod',
    'sqrt_recip_alphas_cumprod', 'sqrt_recipm1_alphas_cumprod', 'posterior_mean_c0_coef',
    'posterior_mean_ct_coef', 'posterior_var', 'posterior_logvar', 'log_alphas_v', 'log_one_minus_alphas_v',
    'log_alphas_cumprod_v', 'log_one_minus_alphas_cumprod_v',
]


def _mlp_spec(prefix, in_dim, out_dim, hidden):
    return [
        (prefix + '.net.0.weight', (hidden, in_dim), 'lin_w'), (prefix + '.net.0.bias', (hidden,), 'lin_b:%d' % in_dim),
        (prefix + '.net.1.weight', (hidden,), 'ln_w'), (prefix + '.net.1.bias', (hidden,), 'ln_b'),
        (prefix + '.net.3.weight', (out_dim, hidden), 'lin_w'), (prefix + '.net.3.bias', (out_dim,), 'lin_b:%d' % hidden),
    ]


def _att_layer_spec(prefix, cfg, num_x2h, num_h2x):
    """reference models/uni_transformer.py:11-40,86-106,143-179 (module order = state_dict order)"""
    H, nh, ng = cfg['hidden_dim'], cfg['n_heads'], cfg['num_r_gaussian']
    r_dim = 4 * ng
    kv_in = 2 * H + cfg['edge_feat_dim'] + r_dim
    ew = cfg['ew_net_type']
    spec = [(prefix + '.distance_expansion.offset', (20,), 'offset')]
    for i in range(num_x2h):
        p = '%s.x2h_layers.%d' % (prefix, i)
        spec += _mlp_spec(p + '.hk_func', kv_in, H, H) + _mlp_spec(p + '.hv_func', kv_in, H, H) + _mlp_spec(p + '.hq_func', H, H, H)
        if ew in ('r', 'm'):
            d = r_dim if ew == 'r' else H
            spec += [(p + '.ew_net.0.weight', (1, d), 'lin_w'), (p + '.ew_net.0.bias', (1,), 'lin_b:%d' % d)]
        if cfg['x2h_out_fc']:
            spec += _mlp_spec(p + '.node_output', 2 * H, H, H)
    for i in range(num_h2x):
        p = '%s.h2x_layers.%d' % (prefix, i)
        spec += _mlp_spec(p + '.xk_func', kv_in, H, H) + _mlp_spec(p + '.xv_func', kv_in, nh, H) + _mlp_spec(p + '.xq_func', H, H, H)
        if ew == 'r':
            spec += [(p + '.ew_net.0.weight', (1, r_dim), 'lin_w'), (p + '.ew_net.0.bias', (1,), 'lin_b:%d' % r_dim)]
    return spec


def state_dict_spec(cfg=None, protein_dim=PROTEIN_FEATURE_DIM, ligand_dim=LIGAND_NUM_CLASSES):
    """Ordered (key, shape, kind) list == the reference module's state_dict() for the default config."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    T, H = cfg['num_diffusion_timesteps'], cfg['hidden_dim']
    emb = H - 1 if cfg['node_indicator'] else H
    spec = [(k, (T,), 'schedule') for k in SCHEDULE_KEYS]
    spec += [('Lt_history', (T,), 'zeros'), ('Lt_count', (T,), 'zeros')]
    spec += [('protein_atom_emb.weight', (emb, protein_dim), 'lin_w'), ('protein_atom_emb.bias', (emb,), 'lin_b:%d' % protein_dim)]
    lig_in = ligand_dim + (0 if cfg['time_emb_dim'] == 0 else 1 if cfg['time_emb_mode'] == 'simple' else cfg['time_emb_dim'])
    spec += [('ligand_atom_emb.weight', (emb, lig_in), 'lin_w'), ('ligand_atom_emb.bias', (emb,), 'lin_b:%d' % lig_in)]
    spec += [('refine_net.distance_expansion.offset', (20,), 'offset')]
    if cfg['ew_net_type'] == 'global':
        spec += _mlp_spec('refine_net.edge_pred_layer', cfg['num_r_gaussian'], 1, H)
    spec += _att_layer_spec('refine_net.init_h_emb_layer', cfg, 1, 0)   # dead weights, strict load needs them
    for l in range(cfg['num_layers']):
        spec += _att_layer_spec('refine_net.base_block.%d' % l, cfg, cfg['num_x2h'], cfg['num_h2x'])
    spec += [('v_inference.0.weight', (H, H), 'lin_w'), ('v_inference.0.bias', (H,), 'lin_b:%d' % H),
             ('v_inference.2.weight', (ligand_dim, H), 'lin_w'), ('v_inference.2.bias', (ligand_dim,), 'lin_b:%d' % H)]
    return spec


def make_state_dict(seed=0, cfg=None, schedules=None, gain=1.0):
    """Deterministic weights.  Linear: U(-1/sqrt(in), 1/sqrt(in))*gain (nn.Linear's default bound);
    LayerNorm: weight 1+0.1*N(0,1), bias 0.1*N(0,1) (non-trivial affine on purpose).
    `schedules`: dict of the 15 fp32 tables (oracle.restate.make_schedules) -- required."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, shape, kind in state_dict_spec(cfg):
        if kind == 'schedule':
            sd[key] = schedules[key].clone()
        elif kind == 'zeros':
            sd[key] = torch.zeros(shape)
        elif kind == 'offset':
            sd[key] = torch.tensor(GAUSSIAN_OFFSETS, dtype=torch.float32)
        elif kind == 'lin_w':
            b = gain / math.sqrt(shape[1])
            sd[key] = (torch.rand(shape, generator=g) * 2 - 1) * b
        elif kind.startswith('lin_b'):
            b = gain / math.sqrt(int(kind.split(':')[1]))
            sd[key] = (torch.rand(shape, generator=g) * 2 - 1) * b
        elif kind == 'ln_w':
            sd[key] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif kind == 'ln_b':
            sd[key] = 0.1 * torch.randn(shape, generator=g)
        else:
            raise ValueError(kind)
    return sd


def make_pocket(seed, n_protein=300, radius=None, min_sep=1.2, cavity=4.0, center=None):
    """One synthetic pocket: positions [n,3] fp32 and one-hot features [n,27] fp32 (SURVEY.md 8(d))."""
    rng = np.random.RandomState(seed)
    if radius is None:
        radius = 12.0 * (n_protein / 300.0) ** (1.0 / 3.0)
    pts = np.zeros((0, 3))
    while len(pts) < n_protein:
        cand = rng.uniform(-radius, radius, size=(4 * n_protein, 3))
        r = np.linalg.norm(cand, axis=1)
        cand = cand[(r <= radius) & (r >= cavity)]
        for c in cand:
            if len(pts) == 0 or np.min(np.sum((pts - c) ** 2, axis=1)) >= min_sep ** 2:
                pts = np.vstack([pts, c[None]])
                if len(pts) == n_protein:
                    break
    if center is None:
        center = rng.uniform(-30.0, 30.0, size=(1, 3))      # pockets live at arbitrary lab-frame offsets
    pos = (pts + center).astype(np.float32)
    elem = rng.choice(6, size=n_protein, p=[0.0, 0.654, 0.152, 0.190, 0.004, 0.0])   # H,C,N,O,S,Se (1h36 freq.)
    aa = rng.randint(0, 20, size=n_protein)
    bb = (rng.uniform(size=n_protein) < 0.45)
    feat = np.zeros((n_protein, PROTEIN_FEATURE_DIM), dtype=np.float32)
    feat[np.arange(n_protein), elem] = 1.0
    feat[np.arange(n_protein), 6 + aa] = 1.0
    feat[:, 26] = bb
    return torch.from_numpy(pos), torch.from_numpy(feat)


def make_batch(seed, n_graphs, n_protein=300, n_ligand=20, distinct_pockets=None, ligand_sizes=None):
    """Batch in the reference's calling convention (scripts/sample_diffusion.py:42-70):
    protein_pos [Np,3], protein_v [Np,27], batch_protein [Np] i64, init_ligand_pos [Nl,3],
    init_ligand_v [Nl] i64, batch_ligand [Nl] i64.  `distinct_pockets` pockets are cycled over graphs."""
    distinct_pockets = distinct_pockets or n_graphs
    pockets = [make_pocket(seed * 1000 + p, n_protein) for p in range(distinct_pockets)]
    g = torch.Generator().manual_seed(seed + 17)
    if ligand_sizes is None:
        ligand_sizes = [n_ligand] * n_graphs
    ppos, pfeat, bp, bl, lpos = [], [], [], [], []
    for i in range(n_graphs):
        pos, feat = pockets[i % distinct_pockets]
        ppos.append(pos); pfeat.append(feat)
        bp.append(torch.full((pos.shape[0],), i, dtype=torch.long))
        bl.append(torch.full((ligand_sizes[i],), i, dtype=torch.long))
        ctr = pos.mean(0, keepdim=True)
        lpos.append(ctr + torch.randn(ligand_sizes[i], 3, generator=g))
    nl = sum(ligand_sizes)
    lig_v = torch.randint(0, LIGAND_NUM_CLASSES, (nl,), generator=g)
    return dict(protein_pos=torch.cat(ppos), protein_v=torch.cat(pfeat), batch_protein=torch.cat(bp),
                init_ligand_pos=torch.cat(lpos), init_ligand_v=lig_v, batch_ligand=torch.cat(bl))


def make_tape(seed, num_steps, n_ligand_atoms, num_classes=LIGAND_NUM_CLASSES):
    """Noise tape in the reference's draw order (models/molopt_score_model.py:677-679 then :685/:161)."""
    g = torch.Generator().manual_seed(seed)
    pos_noise = torch.randn(num_steps, n_ligand_atoms, 3, generator=g)
    v_uniform = torch.rand(num_steps, n_ligand_atoms, num_classes, generator=g)
    return pos_noise, v_uniform
