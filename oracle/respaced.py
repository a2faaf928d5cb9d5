"""Respaced sampling restated on the CPU (TEST INFRASTRUCTURE: float64 Python for the jump tables, torch-CPU fp32 for the chain).

An extension beyond the reference (DESIGN.md section 1).  A time sequence tau_0 > tau_1 > ... > tau_{S-1} >= 0 with tau_0 = T - 1 runs S
steps: step s evaluates the network at t = tau_s, exactly as the reference does at t, and moves the state to p = tau_{s+1}, or to
p = tau_{S-1} - 1 at the last step (the reference's own step at tau_{S-1}; the decoder step when tau_{S-1} = 0).  Unit steps (p = t - 1)
use the checkpoint's tables at t; jump steps (p < t - 1) the exact jump posteriors q(x_p | x_t, x0), q(v_p | v_t, v0), whose coefficients
`jump_coefficients` computes in float64 from the fp32 state-dict tables and `jump_tables` rounds to fp32 once.

Everything else is made of `oracle.restate`'s pinned pieces (the forward network, q_pos_posterior, q_v_pred, the Gumbel-max draw) and
`oracle.fixed_atoms.forward_sample`.  With a unit sequence, `sample_diffusion` is `restate.sample_diffusion` (with a fixed set,
`fixed_atoms.sample_diffusion`) bit for bit (tests/test_respaced.py).  `jump_step` is one step of a respaced chain at any precision,
on `oracle.stepwise.step`, for comparing the engine's steps with float64.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import fixed_atoms, restate, stepwise
from .synth import DEFAULT_MODEL_CONFIG


def targets(time_seq):
    """[(t, p)] of every step of `time_seq`: p = tau_{s+1}, or tau_{S-1} - 1 at the last step."""
    seq = [int(x) for x in time_seq]
    return [(t, seq[s + 1] if s + 1 < len(seq) else t - 1) for s, t in enumerate(seq)]


def prefix_sums(sd):
    """float64 lists over i = 0..t of log(1 - betas[i]) (log alphas_cumprod[t]) and of log_alphas_v[i], summed in order from the fp32
    tables.  1 - abar is taken as -expm1 of the first: from fp32 alphas_cumprod it would keep almost no bits near t = 0."""
    out = []
    for vals in ([math.log1p(-float(b)) for b in sd['betas'].tolist()], [float(x) for x in sd['log_alphas_v'].tolist()]):
        acc, cum = 0.0, []
        for v in vals:
            acc += v
            cum.append(acc)
        out.append(cum)
    return out


def jump_coefficients(sd, t, p, sums=None):
    """float64 coefficients of the jump t -> p (0 <= p < t): with abar = alphas_cumprod and a = abar_t / abar_p,
      c0 = sqrt(abar_p) (1 - a) / (1 - abar_t),  ct = sqrt(a) (1 - abar_p) / (1 - abar_t),  var = (1 - abar_p) (1 - a) / (1 - abar_t),
      lam = sum_{i = p+1..t} log_alphas_v[i] (the log of the type schedule's transition probability from p to t),
      l1ma = log(1 - e^lam + 1e-40)  (the reference's log_1_min_a, models/molopt_score_model.py:169-170).
    Also abar_t, abar_p, 1 - abar_t, 1 - abar_p ('om_t', 'om_p') and logvar = log(var).  With p = t - 1 these are the checkpoint's
    one-step tables at t up to rounding."""
    la, lv = sums if sums is not None else prefix_sums(sd)
    lt, lp = la[t], la[p]
    om_t, om_p, om_a = -math.expm1(lt), -math.expm1(lp), -math.expm1(lt - lp)
    lam = lv[t] - lv[p]
    var = om_p * om_a / om_t
    return {'c0': math.sqrt(math.exp(lp)) * om_a / om_t, 'ct': math.sqrt(math.exp(lt - lp)) * om_p / om_t, 'var': var,
            'logvar': math.log(var), 'lam': lam, 'l1ma': math.log(1.0 - math.exp(lam) + 1e-40), 'ac_t': math.exp(lt), 'ac_p': math.exp(lp),
            'om_t': om_t, 'om_p': om_p}


def jump_tables(sd, time_seq):
    """Per-step tables of a respaced chain, as the engine builds them: 't', 'p' int64 [S], and fp32 [S] 'c0', 'ct', 'logvar', 'la',
    'l1ma'.  Unit steps take the checkpoint's posterior_mean_c0_coef, posterior_mean_ct_coef, posterior_logvar, log_alphas_v and
    log_one_minus_alphas_v at t; jump steps `jump_coefficients` rounded to fp32 once."""
    tp = targets(time_seq)
    sums = prefix_sums(sd)
    unit = ('posterior_mean_c0_coef', 'posterior_mean_ct_coef', 'posterior_logvar', 'log_alphas_v', 'log_one_minus_alphas_v')
    keys = ('c0', 'ct', 'logvar', 'lam', 'l1ma')
    cols = {k: np.zeros(len(tp), np.float32) for k in keys}
    for s, (t, p) in enumerate(tp):
        if p == t - 1:
            for k, name in zip(keys, unit):
                cols[k][s] = sd[name][t].item()
        else:
            c = jump_coefficients(sd, t, p, sums)
            for k in keys:
                cols[k][s] = np.float32(c[k])
    return {'t': np.array([t for t, _ in tp], np.int64), 'p': np.array([p for _, p in tp], np.int64), 'c0': cols['c0'], 'ct': cols['ct'],
            'logvar': cols['logvar'], 'la': cols['lam'], 'l1ma': cols['l1ma']}


def jump_step(sd, cfg, tables, s, xt, vt, x0, logits, pos_noise, v_uniform, pos_only=False, dtype=torch.float32):
    """Step s of a respaced chain, from t = tables['t'][s] to p = tables['p'][s] (`tables` from `jump_tables`), at any precision:
    stepwise.step at t with the entries it reads replaced by the jump's -- posterior_mean_c0_coef, posterior_mean_ct_coef,
    posterior_logvar, log_alphas_v and log_one_minus_alphas_v at t by the step's fp32 coefficients, and the type schedule's cumprod
    tables at t - 1 by those at p.  On a unit step (p = t - 1) nothing is replaced and it is stepwise.step.  Same outputs as
    stepwise.step; with dtype=torch.float64 the fp32 coefficients are read in float64, so the comparison measures the epilogue's
    rounding alone."""
    t, p = int(tables['t'][s]), int(tables['p'][s])
    sdj = {k: sd[k].clone() for k in stepwise.TABLES}
    for name, key in (('posterior_mean_c0_coef', 'c0'), ('posterior_mean_ct_coef', 'ct'), ('posterior_logvar', 'logvar'),
                      ('log_alphas_v', 'la'), ('log_one_minus_alphas_v', 'l1ma')):
        sdj[name][t] = float(tables[key][s])
    if t > 0:
        for name in ('log_alphas_cumprod_v', 'log_one_minus_alphas_cumprod_v'):
            sdj[name][t - 1] = sd[name][max(p, 0)]
    return stepwise.step(sdj, cfg, t, xt, vt, x0, logits, pos_noise, v_uniform, pos_only=pos_only, dtype=dtype)


def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand, pos_noise, v_uniform,
                     time_seq, center_pos_mode='protein', pos_only=False, fixed_mask=None, fixed_tape=None, step_callback=None):
    """The respaced chain on a noise tape pos_noise [S,Nl,3], v_uniform [S,Nl,K]: restate.sample_diffusion's loop
    (models/molopt_score_model.py:633-703) with step s at t = tau_s moving the state to p.  With `fixed_mask` [Nl] bool and the fixed
    tape `fixed_tape` = (pos_noise [S+1,Nl,3], v_uniform [S+1,Nl,K]), the masked rows are held as in fixed_atoms.sample_diffusion, at
    p: a sample of q(x_p | x0_f), q(v_p | v0_f) from tape row s + 1 after step s (x0_f, v0_f themselves when p < 0).
    Returns the reference's dict, trajectories as lists; entry s is the state after step s."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    assert cfg['model_mean_type'] in ('C0', 'noise')
    K = sd['v_inference.2.weight'].shape[0]
    tab = jump_tables(sd, time_seq)
    step_tab = {'posterior_mean_c0_coef': torch.from_numpy(tab['c0']), 'posterior_mean_ct_coef': torch.from_numpy(tab['ct']),
                'posterior_logvar': torch.from_numpy(tab['logvar']), 'log_alphas_v': torch.from_numpy(tab['la']),
                'log_one_minus_alphas_v': torch.from_numpy(tab['l1ma'])}
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, ligand_pos, offset = restate.center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        offset = torch.zeros(num_graphs, 3)
    ligand_v = init_ligand_v
    T = sd['betas'].shape[0]
    if fixed_mask is not None:
        fm = torch.as_tensor(fixed_mask, dtype=torch.bool)
        fpn, fvu = fixed_tape
        x0f, v0f, bf = ligand_pos[fm].clone(), ligand_v[fm].clone(), batch_ligand[fm]

        def hold(pos, v, d, tm):
            pos, v = pos.clone(), v.clone()
            pos[fm], v[fm] = fixed_atoms.forward_sample(sd, x0f, v0f, bf, tm, fpn[d][fm], fvu[d][fm], K, pos_only)
            return pos, v

        ligand_pos, ligand_v = hold(ligand_pos, ligand_v, 0, T - 1)
    pos_traj, v_traj, v0_traj, vt_traj = [], [], [], []
    for s, (i, p) in enumerate(zip(tab['t'].tolist(), tab['p'].tolist())):
        t = torch.full((num_graphs,), i, dtype=torch.long)
        ts = torch.full((num_graphs,), s, dtype=torch.long)                              # index into the per-step tables
        preds = restate.forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step=t)
        pos0, v0 = preds['pred_ligand_pos'], preds['pred_ligand_v']
        if cfg['model_mean_type'] == 'noise':
            eps = pos0 - ligand_pos
            pos0 = restate.extract(sd['sqrt_recip_alphas_cumprod'], t, batch_ligand) * ligand_pos - \
                restate.extract(sd['sqrt_recipm1_alphas_cumprod'], t, batch_ligand) * eps
        pos_mean = restate.q_pos_posterior(step_tab, pos0, ligand_pos, ts, batch_ligand)
        logvar = restate.extract(step_tab['posterior_logvar'], ts, batch_ligand)
        nonzero = (1 - (t == 0).float())[batch_ligand].unsqueeze(-1)
        ligand_pos = pos_mean + nonzero * (0.5 * logvar).exp() * pos_noise[s]
        if not pos_only:
            log_v_recon = F.log_softmax(v0, dim=-1)
            log_v = restate.index_to_log_onehot(ligand_v, K)
            tm1 = torch.full((num_graphs,), max(p, 0), dtype=torch.long)                 # q_v_posterior (:401-409) with t - 1 -> p
            un = restate.q_v_pred(sd, log_v_recon, tm1, batch_ligand, K) + \
                restate.q_v_pred_one_timestep(step_tab, log_v, ts, batch_ligand, K)
            log_model_prob = un - torch.logsumexp(un, dim=-1, keepdim=True)
            ligand_v = restate.log_sample_categorical_from_uniform(log_model_prob, v_uniform[s])
            v0_traj.append(log_v_recon.clone()); vt_traj.append(log_model_prob.clone())
        if fixed_mask is not None:
            ligand_pos, ligand_v = hold(ligand_pos, ligand_v, s + 1, p)
        pos_traj.append((ligand_pos + offset[batch_ligand]).clone())
        v_traj.append(ligand_v.clone())
        if step_callback is not None:
            step_callback(s, i, preds, ligand_pos, ligand_v)
    return {'pos': ligand_pos + offset[batch_ligand], 'v': ligand_v, 'pos_traj': pos_traj, 'v_traj': v_traj,
            'v0_traj': v0_traj, 'vt_traj': vt_traj}


def sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, time_seq, batch_size=16,
                            center_pos_mode='protein', sample_num_atoms='prior', fixed_ligand=None):
    """The rng='cpu' driver (targetdiff_b200.sampling.sample_diffusion_ligand; restate.sample_diffusion_ligand) on a time sequence of S
    steps: per batch the size draws, randn(center), rand(uniform logits), then S steps of randn(Nl, 3) / rand(Nl, K) interleaved, then
    with a fragment `fixed_ligand` = (pos [n_f,3], v [n_f]) the fixed tape's randn(S+1, Nl, 3), rand(S+1, Nl, K) (fixed_atoms' driver).
    Returns the reference's 7-tuple; the time list holds zeros."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    S = len(time_seq)
    n_f = 0
    if fixed_ligand is not None:
        frag_pos, frag_v = torch.as_tensor(fixed_ligand[0]).float(), torch.as_tensor(fixed_ligand[1]).long()
        n_f = len(frag_v)
    all_pos, all_v, all_pos_traj, all_v_traj, all_v0_traj, all_vt_traj, time_list = [], [], [], [], [], [], []
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
        r = sample_diffusion(sd, c, ppos, pfeat, batch_protein, init_pos, init_v, batch_ligand, pn, vu, time_seq,
                             center_pos_mode=center_pos_mode, **fixed)
        cum = np.cumsum([0] + sizes)
        pos = r['pos'].numpy().astype(np.float64)
        all_pos += [pos[cum[k]:cum[k + 1]] for k in range(n_data)]
        ptraj = torch.stack(r['pos_traj']).numpy().astype(np.float64)
        all_pos_traj += [ptraj[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        v = r['v'].numpy()
        all_v += [v[cum[k]:cum[k + 1]] for k in range(n_data)]
        vtraj = torch.stack(r['v_traj']).numpy()
        all_v_traj += [vtraj[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        v0 = torch.stack(r['v0_traj']).numpy()
        vt = torch.stack(r['vt_traj']).numpy()
        all_v0_traj += [v0[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        all_vt_traj += [vt[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        time_list.append(0.0)
        current_i += n_data
    return all_pos, all_v, all_pos_traj, all_v_traj, all_v0_traj, all_vt_traj, time_list
