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


def make_state_dict(seed=0, cfg=None, schedules=None, gain=1.0, ligand_dim=LIGAND_NUM_CLASSES):
    """Deterministic weights.  Linear: U(-1/sqrt(in), 1/sqrt(in))*gain (nn.Linear's default bound);
    LayerNorm: weight 1+0.1*N(0,1), bias 0.1*N(0,1) (non-trivial affine on purpose).
    `schedules`: dict of the 15 fp32 tables (oracle.restate.make_schedules) -- required.
    `ligand_dim`: the ligand class count K (8 'basic', 13 'add_aromatic', 23 'full'); the draws follow the key order, so the
    default K = 13 gives the same weights as before the keyword existed."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, shape, kind in state_dict_spec(cfg, ligand_dim=ligand_dim):
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


def make_batch(seed, n_graphs, n_protein=300, n_ligand=20, distinct_pockets=None, ligand_sizes=None, num_classes=LIGAND_NUM_CLASSES):
    """Batch in the reference's calling convention (scripts/sample_diffusion.py:42-70):
    protein_pos [Np,3], protein_v [Np,27], batch_protein [Np] i64, init_ligand_pos [Nl,3],
    init_ligand_v [Nl] i64 in 0..num_classes-1, batch_ligand [Nl] i64.  `distinct_pockets` pockets are cycled over graphs."""
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
    lig_v = torch.randint(0, num_classes, (nl,), generator=g)
    return dict(protein_pos=torch.cat(ppos), protein_v=torch.cat(pfeat), batch_protein=torch.cat(bp),
                init_ligand_pos=torch.cat(lpos), init_ligand_v=lig_v, batch_ligand=torch.cat(bl))


def _protein_features(rng, n):
    elem = rng.choice(6, size=n, p=[0.0, 0.654, 0.152, 0.190, 0.004, 0.0])
    feat = np.zeros((n, PROTEIN_FEATURE_DIM), dtype=np.float32)
    feat[np.arange(n), elem] = 1.0
    feat[np.arange(n), 6 + rng.randint(0, 20, size=n)] = 1.0
    feat[:, 26] = rng.uniform(size=n) < 0.45
    return torch.from_numpy(feat)


def batch_from_graphs(graphs, seed=0, num_classes=LIGAND_NUM_CLASSES):
    """A batch in make_batch's layout from per-graph (protein_pos [np,3], ligand_pos [nl,3]) pairs (either may be empty): protein
    features and ligand types drawn from `seed`."""
    rng = np.random.RandomState(seed)
    ppos, pfeat, bp, bl, lpos = [], [], [], [], []
    for i, (p, l) in enumerate(graphs):
        p, l = torch.as_tensor(p, dtype=torch.float32).view(-1, 3), torch.as_tensor(l, dtype=torch.float32).view(-1, 3)
        ppos.append(p); pfeat.append(_protein_features(rng, len(p))); lpos.append(l)
        bp.append(torch.full((len(p),), i, dtype=torch.long)); bl.append(torch.full((len(l),), i, dtype=torch.long))
    lig_v = torch.from_numpy(rng.randint(0, num_classes, size=sum(len(l) for l in lpos))).long()
    return dict(protein_pos=torch.cat(ppos), protein_v=torch.cat(pfeat), batch_protein=torch.cat(bp),
                init_ligand_pos=torch.cat(lpos), init_ligand_v=lig_v, batch_ligand=torch.cat(bl))


# ---------------------------------------------------------------------------------------------------------------------------
# Geometry where k-NN selections are decided by ties (tests/test_gpu_graph_geometry.py).  make_batch's random pockets put no two
# squared distances of a row within an ulp of each other, so none of these reach its draws.
# ---------------------------------------------------------------------------------------------------------------------------
LATTICE = 1.5          # exactly representable, as are its multiples and halves: squared distances are exact multiples of 0.5625


def lattice_pocket(seed, n_protein, origin=(3.0, -4.5, 1.5), n_dup=0):
    """`n_protein` sites of a cubic lattice of spacing LATTICE around `origin` (a lattice point): the ones nearest the origin in a
    seeded shuffled order, so each row has many exactly equal squared distances.  The last `n_dup` atoms repeat earlier sites (a
    duplicate then always has a coincident atom of smaller index)."""
    rng = np.random.RandomState(seed)
    m = int(np.ceil((n_protein + 8) ** (1.0 / 3.0) / 2.0)) + 2
    g = np.arange(-m, m + 1)
    sites = np.stack(np.meshgrid(g, g, g, indexing='ij'), -1).reshape(-1, 3)
    r2 = (sites ** 2).sum(1)
    sites = sites[np.argsort(r2 + rng.uniform(0, 0.5, size=len(r2)), kind='stable')][:n_protein - n_dup]
    sites = sites[rng.permutation(len(sites))]
    if n_dup:
        sites = np.concatenate([sites, sites[rng.choice(len(sites), n_dup, replace=False)]])
    return (sites * LATTICE + np.asarray(origin)).astype(np.float32)


def tie_ligand(seed, protein_pos, n_site=4, n_half=6, n_pairs=3, origin=(3.0, -4.5, 1.5)):
    """Ligand atoms for a lattice pocket: `n_site` on protein sites (d = 0 to a protein atom), `n_half` on half-lattice points
    (equidistant from 2, 4 or 8 sites), and `n_pairs` coincident ligand pairs (each on a half-lattice point)."""
    rng = np.random.RandomState(seed)
    on_site = protein_pos[rng.choice(len(protein_pos), n_site, replace=False)]
    half = []
    for i in range(n_half + n_pairs):
        c = rng.randint(-2, 3, size=3).astype(np.float64)
        c[rng.permutation(3)[:1 + i % 3]] += 0.5                  # 1, 2 or 3 half-integer coordinates
        half.append(c * LATTICE + np.asarray(origin))
    half = np.asarray(half, dtype=np.float32)
    pairs = np.repeat(half[n_half:], 2, axis=0)
    return np.concatenate([on_site, half[:n_half], pairs]).astype(np.float32)


def d2_fp32(a, b):
    """The canonical k-NN distance key (SURVEY.md Appendix A.3) of every row of `a` [n,3] against every row of `b` [m,3]:
    ((dx*dx)+(dy*dy))+(dz*dz) with dx = a - b and every op rounded to fp32 (no FMA contraction).  numpy float32 [n,m]."""
    f32 = np.float32
    a, b = np.asarray(a, dtype=f32).reshape(-1, 3), np.asarray(b, dtype=f32).reshape(-1, 3)
    dx, dy, dz = (a[:, None, i] - b[None, :, i] for i in range(3))
    return ((dx * dx).astype(f32) + (dy * dy).astype(f32)).astype(f32) + (dz * dz).astype(f32)


def _d2_orders(q, a, b):
    """For candidates a (smaller index) and b of query q: is a before b under the canonical fp32 key, under the two FMA-contracted
    evaluations of d2 nvcc can form, and under exact d2?"""
    from fractions import Fraction
    f32 = np.float32
    d = [[f32(f32(c[i]) - f32(q[i])) for i in range(3)] for c in (a, b)]
    canon = d2_fp32(q, np.stack([a, b]))[0]

    def fma(x, y, z):
        return f32(float(Fraction(float(x)) * Fraction(float(x if y is None else y)) + Fraction(float(z))))

    def fma1(v):                                   # fma(dz, dz, fma(dy, dy, dx * dx))
        return fma(v[2], None, fma(v[1], None, f32(v[0] * v[0])))

    def fma2(v):                                   # fma(dz, dz, fma(dx, dx, dy * dy))
        return fma(v[2], None, fma(v[0], None, f32(v[1] * v[1])))

    def exact(v):
        return sum(Fraction(float(x)) ** 2 for x in v)

    return [(canon[0], 0) < (canon[1], 1)] + [(f(d[0]), 0) < (f(d[1]), 1) for f in (fma1, fma2, exact)]


def near_tie_triple(rng, centre, r=1.6):
    """A (q, a, b) triple found by a seeded search: q within 1 A of `centre`, a and b about `r` from q, a before b (a taking the
    smaller index) under the canonical fp32 key but not under either FMA-contracted d2, nor under exact d2."""
    while True:
        q = (rng.uniform(-1, 1, 3) + centre).astype(np.float32)
        v = rng.normal(size=3)
        a = (q + v / np.linalg.norm(v) * r).astype(np.float32)
        b = a.copy()
        for i in range(3):
            b[i] = np.nextafter(b[i], np.float32(np.inf) if rng.uniform() < 0.5 else np.float32(-np.inf))
        o = _d2_orders(q, a, b)
        if o[0] and not o[1] and not o[2] and not o[3]:
            return q, a, b


def near_tie_graph(seed, n_triples=24, n_fill=60, spacing=7.0, frame=20.0):
    """One graph of near-tie triples, one per cell of a grid of `spacing` about `frame` A from the origin (where coordinate
    differences round; each q's nearest atoms are its a and b), in four roles: q ligand with a, b protein; q protein with a, b
    ligand; all three ligand; all three protein (the pair then sits in q's cached protein keys).  `n_fill` protein atoms far from the
    cells keep np above k.  Returns (protein_pos, ligand_pos)."""
    rng = np.random.RandomState(seed)
    prot, lig = [], []
    for i in range(n_triples):
        centre = np.array([i % 4, (i // 4) % 4, i // 16], dtype=np.float64) * spacing + frame
        q, a, b = near_tie_triple(rng, centre)
        role = i % 4
        if role == 0:
            lig.append(q); prot += [a, b]
        elif role == 1:
            prot.append(q); lig += [a, b]
        elif role == 2:
            lig += [q, a, b]
        else:
            prot += [q, a, b]
    fill = rng.uniform(-1, 1, size=(n_fill, 3)) * 6.0 - 40.0
    return np.concatenate([np.asarray(prot), fill]).astype(np.float32), np.asarray(lig, dtype=np.float32)


def hybrid_norm_tie_graph(k, seed=2, n_far=12):
    """One graph where the reference's hybrid graph and the canonical one differ: a ligand atom L, k - 1 protein atoms clearly nearer
    than 3 A, then protein atoms k - 1 and k with equal torch.norm distance to L but d2(k - 1) < d2(k) in fp32, then `n_far`
    farther ones; two more ligand atoms far from the tie.  Returns (protein_pos, ligand_pos)."""
    rng = np.random.RandomState(seed)
    L = np.array([[0.125, -0.375, 0.25]], dtype=np.float32)
    Lt = torch.from_numpy(L)
    pair = None
    while pair is None:
        v = rng.normal(size=3)
        p1 = (L[0] + v / np.linalg.norm(v) * 3.0).astype(np.float32)
        for i in range(3):
            p2 = p1.copy()
            p2[i] = np.nextafter(p1[i], np.float32(np.inf) if rng.uniform() < 0.5 else np.float32(-np.inf))
            P = torch.from_numpy(np.stack([p1, p2]))
            d = torch.norm(Lt.unsqueeze(1) - P.unsqueeze(0), p=2, dim=-1)[0]
            d2 = [float(x) for x in d2_fp32(L, np.stack([p1, p2]))[0]]
            if d[0] == d[1] and d2[0] != d2[1]:
                pair = (p1, p2) if d2[0] < d2[1] else (p2, p1)
                break
    near = []
    while len(near) < k - 1:
        v = rng.normal(size=3)
        near.append(L[0] + v / np.linalg.norm(v) * rng.uniform(1.0, 2.6))
    far = []
    while len(far) < n_far:
        v = rng.normal(size=3)
        far.append(L[0] + v / np.linalg.norm(v) * rng.uniform(3.5, 6.0))
    prot = np.concatenate([np.asarray(near), np.stack(pair), np.asarray(far)]).astype(np.float32)
    lig = np.concatenate([L, L + np.array([[12.0, 0, 0], [0, 12.0, 0]], dtype=np.float32)]).astype(np.float32)
    return prot, lig


def make_ragged_batch(seed, protein_sizes, ligand_sizes, num_classes=LIGAND_NUM_CLASSES):
    """Graphs with their own protein and ligand counts (either may be 0; the reference's scatter_mean has no row for a trailing
    graph without protein atoms, so keep one last).  Pockets as make_pocket, ligand atoms around the pocket centre."""
    g = torch.Generator().manual_seed(seed + 17)
    graphs = []
    for i, (npr, nl) in enumerate(zip(protein_sizes, ligand_sizes)):
        if npr:
            pos, _ = make_pocket(seed * 1000 + i, npr)
            ctr = pos.mean(0, keepdim=True)
        else:
            pos, ctr = torch.zeros(0, 3), torch.rand(1, 3, generator=g) * 40 - 20
        graphs.append((pos, ctr + torch.randn(nl, 3, generator=g)))
    return batch_from_graphs(graphs, seed, num_classes)


def make_tape(seed, num_steps, n_ligand_atoms, num_classes=LIGAND_NUM_CLASSES):
    """Noise tape in the reference's draw order (models/molopt_score_model.py:677-679 then :685/:161)."""
    g = torch.Generator().manual_seed(seed)
    pos_noise = torch.randn(num_steps, n_ligand_atoms, 3, generator=g)
    v_uniform = torch.rand(num_steps, n_ligand_atoms, num_classes, generator=g)
    return pos_noise, v_uniform
