"""Resampled sampling on a time path restated on the CPU (TEST INFRASTRUCTURE: float64 Python for the tables, torch-CPU fp32 for the
chain).

An extension beyond the reference (DESIGN.md section 1; RePaint, Lugmayr et al. 2022).  A time path tau_0, ..., tau_{S-1} starts at
T - 1 (or at a start time), never repeats a time twice in a row and goes down at its first step.  Step s moves the state from
t = tau_s to p = tau_{s+1}, or to tau_{S-1} - 1 at the last step (respaced.targets):
  p < t, a denoising step: oracle.respaced's step (respaced.jump_step), fixed rows resampled at p;
  p > t, a re-noising step: the forward process q(x_p | x_t), q(v_p | v_t) with no network (`renoise_step`), fixed rows resampled at p.
Step s of either kind reads row s of the tapes, and the fixed tape row s + 1, so a path of S steps uses the stream of any S-step chain.

`renoise_coefficients` gives a re-noising step's coefficients in float64 from the prefix sums of oracle.respaced, `path_tables` every
step's fp32 table row as the engine builds it, and `resampled_time_path` the RePaint path (the same function as
targetdiff_b200.sampling.resampled_time_path, restated here so that the oracle does not import the package).  On a strictly decreasing
path `sample_diffusion` is oracle.respaced.sample_diffusion bit for bit (tests/test_resample.py).
"""
import math

import numpy as np
import torch

from . import fixed_atoms, respaced, restate, start_ligand
from .synth import DEFAULT_MODEL_CONFIG


def resampled_time_path(base, resamplings=1, jump_length=1):
    """The RePaint path over the decreasing base sequence b_0 > ... > b_{n-1}: base indices in blocks [k j, e], e = min(k j + j, n - 1);
    each block is denoised from b_{kj} down to b_e, then r - 1 times re-noised in one step back up to b_{kj} and denoised again; the
    path ends with the last step at b_{n-1}."""
    b = [int(x) for x in base]
    r, j, n = int(resamplings), int(jump_length), len(b)
    path = [b[0]]
    for k0 in range(0, n - 1, j):
        e = min(k0 + j, n - 1)
        for rep in range(r):
            if rep > 0:
                path.append(b[k0])
            path += b[k0 + 1:e + 1]
    return path


def renoise_coefficients(sd, t, p, sums=None):
    """float64 coefficients of the re-noising step t -> p (p > t): with r = abar_p / abar_t, log r = sum_{i = t+1..p} log1p(-beta_i),
      c = sqrt(r), d = sqrt(1 - r) (1 - r = -expm1(log r)),
      lam = sum_{i = t+1..p} log_alphas_v[i] (the log of the type schedule's transition probability from t to p),
      l1ma = log(1 - e^lam + 1e-40).
    Also 'r' and 'log_r'."""
    la, lv = sums if sums is not None else respaced.prefix_sums(sd)
    log_r = la[p] - la[t]
    lam = lv[p] - lv[t]
    return {'c': math.sqrt(math.exp(log_r)), 'd': math.sqrt(-math.expm1(log_r)), 'r': math.exp(log_r), 'log_r': log_r, 'lam': lam,
            'l1ma': math.log(1.0 - math.exp(lam) + 1e-40)}


def path_tables(sd, path):
    """Per-step tables of a time path as the engine builds them: 't', 'p' int64 [S] and fp32 [S] 'c0', 'ct', 'logvar', 'la', 'l1ma'.
    Denoising steps as respaced.jump_tables (the checkpoint's tables at t on unit steps, the jump coefficients rounded once otherwise).
    Re-noising steps: c0 <- c, ct <- d, logvar <- 0, la <- lam, l1ma <- l1ma of `renoise_coefficients`, each rounded to fp32 once; on a
    unit step up (p = t + 1) la and l1ma are the checkpoint's log_alphas_v[p] and log_one_minus_alphas_v[p] (the reference's
    q_v_pred_one_timestep, models/molopt_score_model.py:371-381)."""
    tp = respaced.targets(path)
    sums = respaced.prefix_sums(sd)
    keys = ('c0', 'ct', 'logvar', 'la', 'l1ma')
    cols = {k: np.zeros(len(tp), np.float32) for k in keys}
    unit = ('posterior_mean_c0_coef', 'posterior_mean_ct_coef', 'posterior_logvar', 'log_alphas_v', 'log_one_minus_alphas_v')
    for s, (t, p) in enumerate(tp):
        if p > t:
            c = renoise_coefficients(sd, t, p, sums)
            row = [c['c'], c['d'], 0.0, c['lam'], c['l1ma']]
            if p == t + 1:
                row[3:] = [sd['log_alphas_v'][p].item(), sd['log_one_minus_alphas_v'][p].item()]
        elif p == t - 1:
            row = [sd[name][t].item() for name in unit]
        else:
            c = respaced.jump_coefficients(sd, t, p, sums)
            row = [c['c0'], c['ct'], c['logvar'], c['lam'], c['l1ma']]
        for k, x in zip(keys, row):
            cols[k][s] = np.float32(x)
    return dict(t=np.array([t for t, _ in tp], np.int64), p=np.array([p for _, p in tp], np.int64), **cols)


def renoise_step(sd, tables, s, xt, vt, pos_noise, v_uniform, K, pos_only=False, dtype=torch.float32):
    """Re-noising step s of a time path (tables['p'][s] > tables['t'][s]) for every row, from x_t [n,3], v_t [n] and the step's normals
    [n,3] / uniforms [n,K].  fp32 (default): the kernel's roundings -- c and d from `tables` (fp32), x_p = c x_t + d eps with each
    product and the sum rounded once; log q(v_p | v_t) = log_add_exp(log_onehot(v_t) + la, l1ma - log K) in fp32, the type by Gumbel-max
    over it (q_v_sample's form, models/molopt_score_model.py:394-398).  float64: the same from `renoise_coefficients` in float64, not
    rounded.  Returns {'pos', 'v', 'vt' (normalised log q, None with pos_only), 'margin' (best Gumbel score minus the runner-up),
    'scale' (|c x_t| + |d eps|, the position's magnitude for relative errors)}; with pos_only the types are v_t."""
    t, p = int(tables['t'][s]), int(tables['p'][s])
    if dtype == torch.float64:
        c = renoise_coefficients(sd, t, p)
        cc, dd, la, l1ma = c['c'], c['d'], c['lam'], c['l1ma']
    else:
        cc, dd, la, l1ma = (float(tables[k][s]) for k in ('c0', 'ct', 'la', 'l1ma'))
    one = torch.ones((), dtype=dtype)
    cc, dd, la, l1ma = cc * one, dd * one, la * one, l1ma * one
    x, eps = xt.to(dtype), pos_noise.to(dtype)
    pos = cc * x + dd * eps
    out = {'pos': pos, 'v': vt.clone(), 'vt': None, 'margin': None, 'scale': (cc * x).abs() + (dd * eps).abs()}
    if pos_only:
        return out
    log_oh = restate.index_to_log_onehot(vt, K).to(dtype)
    lq = restate.log_add_exp(log_oh + la, (l1ma - np.log(K)) * torch.ones(1, dtype=dtype))
    score = -torch.log(-torch.log(v_uniform.to(dtype) + 1e-30) + 1e-30) + lq
    top2 = score.topk(2, dim=-1).values
    out.update(v=restate.log_sample_categorical_from_uniform(lq, v_uniform.to(dtype)), vt=lq - torch.logsumexp(lq, dim=-1, keepdim=True),
               margin=top2[:, 0] - top2[:, 1])
    return out


def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand, pos_noise, v_uniform,
                     time_path, center_pos_mode='protein', pos_only=False, fixed_mask=None, fixed_tape=None, start_time=None,
                     start_tape=None, step_callback=None):
    """The chain on a time path on the noise tape pos_noise [S,Nl,3], v_uniform [S,Nl,K]; with `fixed_mask` [Nl] bool the rows held to
    the forward process of their initial rows on the fixed tape (pos_noise [S+1,Nl,3], v_uniform [S+1,Nl,K] or None); with
    `start_time` = t0 the initial ligand is a clean start ligand drawn to t0 first (oracle.start_ligand.start_state, start tape
    (pos_noise [Nl,3], v_uniform [Nl,K] or None)).  Trajectories as lists, entry s the state after step s: after a re-noising step
    v0_traj repeats the entry before and vt_traj holds the normalised log q(v_p | v_t).  Returns the reference's dict."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    T = sd['betas'].shape[0]
    tab = path_tables(sd, time_path)
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, x0, offset = restate.center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        offset = torch.zeros(num_graphs, 3)
    v0 = init_ligand_v.clone()
    fm = None if fixed_mask is None else torch.as_tensor(fixed_mask, dtype=torch.bool)
    if fm is not None and not bool(fm.any()):
        fm = None

    def hold(pos, v, d, tm):
        vu = torch.zeros(len(batch_ligand), K) if fixed_tape[1] is None else fixed_tape[1][d]
        pos, v = pos.clone(), v.clone()
        pos[fm], v[fm] = fixed_atoms.forward_sample(sd, x0[fm], v0[fm], batch_ligand[fm], tm, fixed_tape[0][d][fm], vu[fm], K, pos_only)
        return pos, v

    if start_time is not None:
        ligand_pos, ligand_v = start_ligand.start_state(sd, x0, v0, batch_ligand, int(start_time), start_tape, K, pos_only, fm, fixed_tape)
    else:
        ligand_pos, ligand_v = x0, v0
        if fm is not None:
            ligand_pos, ligand_v = hold(ligand_pos, ligand_v, 0, T - 1)
    pos_traj, v_traj, v0_traj, vt_traj = [], [], [], []
    for s, (t, p) in enumerate(zip(tab['t'].tolist(), tab['p'].tolist())):
        preds = None
        if p < t:
            tt = torch.full((num_graphs,), t, dtype=torch.long)
            preds = restate.forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step=tt)
            out = respaced.jump_step(sd, cfg, tab, s, ligand_pos, ligand_v, preds['pred_ligand_pos'], preds['pred_ligand_v'], pos_noise[s],
                                     v_uniform[s], pos_only=pos_only)
            if not pos_only:
                v0_traj.append(out['v0'].clone())
        else:
            out = renoise_step(sd, tab, s, ligand_pos, ligand_v, pos_noise[s], v_uniform[s], K, pos_only=pos_only)
            if not pos_only:
                v0_traj.append(v0_traj[-1].clone())
        ligand_pos, ligand_v = out['pos'], out['v']
        if not pos_only:
            vt_traj.append(out['vt'].clone())
        if fm is not None:
            ligand_pos, ligand_v = hold(ligand_pos, ligand_v, s + 1, p)
        pos_traj.append((ligand_pos + offset[batch_ligand]).clone())
        v_traj.append(ligand_v.clone())
        if step_callback is not None:
            step_callback(s, t, preds, ligand_pos, ligand_v)
    return {'pos': ligand_pos + offset[batch_ligand], 'v': ligand_v, 'pos_traj': pos_traj, 'v_traj': v_traj,
            'v0_traj': v0_traj, 'vt_traj': vt_traj}


def sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, time_path, batch_size=16,
                            center_pos_mode='protein', sample_num_atoms='prior', fixed_ligand=None):
    """The rng='cpu' driver (targetdiff_b200.sampling.sample_diffusion_ligand) on a time path of S steps, with the draws of
    oracle.respaced's driver for a time sequence of S steps: per batch the size draws, randn(center), rand(uniform logits), S steps of
    randn(Nl, 3) / rand(Nl, K) interleaved, then with a fragment `fixed_ligand` = (pos [n_f,3], v [n_f]) the fixed tape's
    randn(S+1, Nl, 3), rand(S+1, Nl, K).  Returns the reference's 7-tuple; the time list holds zeros."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    S = len(time_path)
    n_f = 0
    if fixed_ligand is not None:
        frag_pos, frag_v = torch.as_tensor(fixed_ligand[0]).float(), torch.as_tensor(fixed_ligand[1]).long()
        n_f = len(frag_v)
    outs = [[] for _ in range(6)]
    num_batch = int(np.ceil(num_samples / batch_size))
    current_i = 0
    n_prot = protein_pos.shape[0]
    for i in range(num_batch):
        n_data = batch_size if i < num_batch - 1 else num_samples - batch_size * (num_batch - 1)
        batch_protein = torch.repeat_interleave(torch.arange(n_data), n_prot)
        ppos = protein_pos.repeat(n_data, 1)
        pfeat = protein_atom_feature.float().repeat(n_data, 1)
        if sample_num_atoms == 'prior':
            pocket_size = restate.get_space_size(protein_pos.detach().cpu().numpy())
            sizes = [int(restate.sample_atom_num(pocket_size, prior)) for _ in range(n_data)]
        elif sample_num_atoms == 'range':
            sizes = list(range(current_i + 1, current_i + n_data + 1))
        else:
            raise ValueError(sample_num_atoms)
        if n_f:
            sizes = [max(n, n_f + 1) for n in sizes]
        batch_ligand = torch.repeat_interleave(torch.arange(n_data), torch.tensor(sizes))
        n_lig = len(batch_ligand)
        s3 = torch.zeros(n_data, 3).index_add_(0, batch_protein, ppos)
        center = s3 / torch.zeros(n_data).index_add_(0, batch_protein, torch.ones(len(batch_protein)))[:, None]
        bc = center[batch_ligand]
        init_pos = bc + torch.randn_like(bc)
        init_v = restate.log_sample_categorical_from_uniform(torch.zeros(n_lig, K), torch.rand(n_lig, K))
        pn = torch.empty(S, n_lig, 3)
        vu = torch.zeros(S, n_lig, K)
        for st in range(S):
            pn[st] = torch.randn(n_lig, 3)
            vu[st] = torch.rand(n_lig, K)
        fixed = {}
        if n_f:
            starts = np.cumsum([0] + sizes[:-1])
            rows = torch.from_numpy((starts[:, None] + np.arange(n_f)[None, :]).reshape(-1))
            mask = torch.zeros(n_lig, dtype=torch.bool)
            mask[rows] = True
            init_pos[rows] = frag_pos.repeat(n_data, 1)
            init_v = init_v.clone()
            init_v[rows] = frag_v.repeat(n_data)
            fixed = {'fixed_mask': mask, 'fixed_tape': (torch.randn(S + 1, n_lig, 3), torch.rand(S + 1, n_lig, K))}
        r = sample_diffusion(sd, c, ppos, pfeat, batch_protein, init_pos, init_v, batch_ligand, pn, vu, time_path,
                             center_pos_mode=center_pos_mode, **fixed)
        cum = np.cumsum([0] + sizes)
        per = [r['pos'].numpy().astype(np.float64), r['v'].numpy(), torch.stack(r['pos_traj']).numpy().astype(np.float64),
               torch.stack(r['v_traj']).numpy(), torch.stack(r['v0_traj']).numpy(), torch.stack(r['vt_traj']).numpy()]
        for j, arr in enumerate(per):
            outs[j] += [arr[cum[k]:cum[k + 1]] if j < 2 else arr[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        current_i += n_data
    return tuple(outs) + ([0.0] * num_batch,)
