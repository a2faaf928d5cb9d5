"""Clash guidance restated on the CPU (TEST INFRASTRUCTURE, torch-CPU at any dtype: float64 for the error tables, fp32 for chains).

An extension beyond the reference (DESIGN.md section 1, "Clash guidance").  At every denoising step, network time t, each ligand atom
a of graph g has the step's x0 prediction y (after the 'noise' mean type's conversion; centred frame).  For each protein atom p of g
at its bound position x_p, r = y - x_p and d = |r|; a pair contributes when 0 < d < rho, and the guided prediction is

    y_hat = y + lambda * sum (rho - d) r / d     over the contributing pairs      (= y - (lambda / 2) grad E(y),
                                                                                      E(y) = sum_p max(0, rho - |y - x_p|)^2)

An atom without a contributing pair keeps y exactly.  The step then runs unchanged with y_hat in place of x0.

`guide` is the rule; `energy` is E (for finite differences); `guided_jump_step` is `oracle.respaced.jump_step` with the hook applied
after the 'noise' reconstruction, by running jump_step in C0 mode on y_hat -- the same operations as the 'noise' mode's step on the
reconstructed x0, since that step reads x0 only through the reconstruction.  `sample_diffusion` is `oracle.resample.sample_diffusion`
(default, respaced, fragment, start and path chains) with a `guidance` hook, and `sample_diffusion_ligand` is
`oracle.resample.sample_diffusion_ligand` (the rng='cpu' driver) on that chain; with guidance=None each is the original itself, and
at strength 0 each gives the original's bits (tests/test_clash_guidance.py).  The existing oracle modules are left as they are.
"""
import numpy as np
import torch

from . import fixed_atoms, resample, respaced, restate, start_ligand
from .layerwise import default_dtype
from .synth import DEFAULT_MODEL_CONFIG


def guide(y, protein_pos, batch_ligand, batch_protein, radius, strength, dtype=torch.float64):
    """The guided prediction [Nl,3] at `dtype` of the x0 predictions y [Nl,3] against the protein atoms (protein_pos [Np,3]) of each
    ligand atom's own graph.  strength == 0: y itself.  Sums run over a graph's protein atoms in order (torch's reduction order at fp32
    is not the engine's: compare fp32 results with a tolerance)."""
    y = y.to(dtype)
    out = y.clone()
    if float(strength) == 0.0:
        return out
    pp = protein_pos.to(dtype)
    rho = torch.tensor(float(radius), dtype=dtype)
    lam = torch.tensor(float(strength), dtype=dtype)
    for g in torch.unique(batch_ligand).tolist():
        rows = (batch_ligand == g).nonzero().reshape(-1)
        p = pp[batch_protein == g]
        if len(p) == 0:
            continue
        r = y[rows][:, None, :] - p[None, :, :]                                  # [na, np, 3]
        d = torch.sqrt((r * r).sum(-1))
        m = (d > 0) & (d < rho)
        w = torch.where(m, (rho - d) / torch.where(m, d, torch.ones_like(d)), torch.zeros_like(d))
        s = (w[..., None] * r).sum(1)
        hit = m.any(1)
        out[rows[hit]] = y[rows[hit]] + lam * s[hit]
    return out


def energy(y, protein_pos, batch_ligand, batch_protein, radius):
    """E(y) = sum over ligand atoms and the protein atoms of their graph of max(0, rho - |y - x_p|)^2, float64."""
    y, pp = y.double(), protein_pos.double()
    d = torch.cdist(y, pp, compute_mode='donot_use_mm_for_euclid_dist')
    same = batch_ligand[:, None] == batch_protein[None, :]
    return float((torch.clamp(float(radius) - d, min=0.0) ** 2 * same).sum())


def hook(radius, strength, dtype=torch.float32):
    """A `guidance` hook for the chains below: (y, protein_pos, batch_ligand, batch_protein) -> guide(...) at `dtype`."""
    return lambda y, pp, bl, bp: guide(y, pp, bl, bp, radius, strength, dtype=dtype)


def x0_prediction(sd, cfg, t, xt, x0, dtype=torch.float32):
    """The step's x0 prediction at time t from the network output x0 [Nl,3] and the state xt: x0 in C0 mode; in 'noise' mode the
    reconstruction of oracle.stepwise.step, op by op (reference models/molopt_score_model.py:419-422,663-666)."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    with default_dtype(dtype):
        xt, x0 = xt.to(dtype), x0.to(dtype)
        if cfg['model_mean_type'] != 'noise':
            return x0
        tt = torch.full((1,), int(t), dtype=torch.long)
        batch = torch.zeros(xt.shape[0], dtype=torch.long)
        sra, srm1 = sd['sqrt_recip_alphas_cumprod'].to(dtype), sd['sqrt_recipm1_alphas_cumprod'].to(dtype)
        eps = x0 - xt
        return restate.extract(sra, tt, batch) * xt - restate.extract(srm1, tt, batch) * eps


def guided_jump_step(sd, cfg, tables, s, xt, vt, x0, logits, pos_noise, v_uniform, guide_fn, pos_only=False, dtype=torch.float32):
    """respaced.jump_step with the x0 prediction replaced by guide_fn(x0 prediction) (guide_fn None: jump_step itself).  Returns
    jump_step's dict plus 'x0' (the prediction) and 'x0_hat' (the guided one)."""
    if guide_fn is None:
        return respaced.jump_step(sd, cfg, tables, s, xt, vt, x0, logits, pos_noise, v_uniform, pos_only=pos_only, dtype=dtype)
    t = int(tables['t'][s])
    y = x0_prediction(sd, cfg, t, xt, x0, dtype=dtype)
    y_hat = guide_fn(y).to(dtype)
    c0 = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    c0['model_mean_type'] = 'C0'
    out = respaced.jump_step(sd, c0, tables, s, xt, vt, y_hat, logits, pos_noise, v_uniform, pos_only=pos_only, dtype=dtype)
    out.update(x0=y, x0_hat=y_hat)
    return out


def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand, pos_noise, v_uniform,
                     time_path, center_pos_mode='protein', pos_only=False, fixed_mask=None, fixed_tape=None, start_time=None,
                     start_tape=None, guidance=None, step_callback=None):
    """oracle.resample.sample_diffusion with clash guidance: `guidance` a hook (y, protein_pos, batch_ligand, batch_protein) -> y_hat
    (e.g. `hook(radius, strength)`), applied at every denoising step to the x0 prediction in the centred frame, with the centred
    protein positions.  guidance=None: resample.sample_diffusion itself.  The loop below is that function's, with
    respaced.jump_step replaced by guided_jump_step."""
    if guidance is None:
        return resample.sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand,
                                         pos_noise, v_uniform, time_path, center_pos_mode=center_pos_mode, pos_only=pos_only,
                                         fixed_mask=fixed_mask, fixed_tape=fixed_tape, start_time=start_time, start_tape=start_tape,
                                         step_callback=step_callback)
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    T = sd['betas'].shape[0]
    tab = resample.path_tables(sd, time_path)
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, x0, offset = restate.center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        offset = torch.zeros(num_graphs, 3)
    v0 = init_ligand_v.clone()
    fm = None if fixed_mask is None else torch.as_tensor(fixed_mask, dtype=torch.bool)
    if fm is not None and not bool(fm.any()):
        fm = None
    guide_fn = lambda y: guidance(y, protein_pos, batch_ligand, batch_protein)

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
            out = guided_jump_step(sd, cfg, tab, s, ligand_pos, ligand_v, preds['pred_ligand_pos'], preds['pred_ligand_v'], pos_noise[s],
                                   v_uniform[s], guide_fn, pos_only=pos_only)
            if not pos_only:
                v0_traj.append(out['v0'].clone())
        else:
            out = resample.renoise_step(sd, tab, s, ligand_pos, ligand_v, pos_noise[s], v_uniform[s], K, pos_only=pos_only)
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


def unit_path(T, num_steps=None):
    """The default chain's time path T - 1, ..., T - num_steps (all T steps by default) as a list."""
    return list(range(T - 1, T - 1 - (T if num_steps is None else int(num_steps)), -1))



def sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, time_path, batch_size=16,
                            center_pos_mode='protein', sample_num_atoms='prior', fixed_ligand=None, guidance=None):
    """oracle.resample.sample_diffusion_ligand (the rng='cpu' driver on a time path) with the chain of `sample_diffusion` above and its
    `guidance` hook; guidance=None: that driver itself.  The draws are that driver's, in its order: guidance draws nothing."""
    if guidance is None:
        return resample.sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, time_path,
                                                batch_size=batch_size, center_pos_mode=center_pos_mode, sample_num_atoms=sample_num_atoms,
                                                fixed_ligand=fixed_ligand)
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
                             center_pos_mode=center_pos_mode, guidance=guidance, **fixed)
        cum = np.cumsum([0] + sizes)
        per = [r['pos'].numpy().astype(np.float64), r['v'].numpy(), torch.stack(r['pos_traj']).numpy().astype(np.float64),
               torch.stack(r['v_traj']).numpy(), torch.stack(r['v0_traj']).numpy(), torch.stack(r['vt_traj']).numpy()]
        for j, arr in enumerate(per):
            outs[j] += [arr[cum[k]:cum[k + 1]] if j < 2 else arr[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        current_i += n_data
    return tuple(outs) + ([0.0] * num_batch,)
