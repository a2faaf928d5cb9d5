"""Element constraints restated on the CPU (TEST INFRASTRUCTURE, torch-CPU at any dtype: float64 for the error tables, fp32 for chains).

An extension beyond the reference (DESIGN.md section 1, "Element constraints").  Each ligand row a has an allowed set A_a of classes
(a [Nl, K] bool mask, no row empty).  At every denoising step:
  1. the type head's log_softmax runs over A_a only: log v0_hat = -inf outside it (the factorised x0 prediction conditioned on
     v0 in A_a), and the posterior runs unchanged on it;
  2. on the decoder step (target time p < 0, which is always the unit step from t = 0) the unnormalised log posterior is -inf outside
     A_a before its normalisation, so that it is renormalised over A_a and the Gumbel-max draw only picks an allowed class.
Intermediate states are drawn from the whole posterior.  Re-noising steps, the start and fixed-row draws ignore the mask.  A mask that
allows every class changes no value: masked_fill writes nothing and the step is the original's, op for op.

`conditioned_step` is `oracle.clash_guidance.guided_jump_step` (so `oracle.respaced.jump_step` without guidance) with that rule;
`sample_diffusion` is `oracle.clash_guidance.sample_diffusion` (default, respaced, fragment, start and path chains, with or without
clash guidance) with an `allowed` mask, and `sample_diffusion_ligand` is `oracle.clash_guidance.sample_diffusion_ligand` (the
rng='cpu' driver) with a set for the free atoms.  With allowed=None each is the original itself, and with the full set each gives the
original's bits (tests/test_type_constraints.py).  The existing oracle modules are left as they are.
"""
import numpy as np
import torch

from . import clash_guidance, fixed_atoms, resample, restate, start_ligand, stepwise
from .layerwise import default_dtype
from .synth import DEFAULT_MODEL_CONFIG


def decoder_types(sd, vt, log_v0, v_uniform, allowed, dtype=torch.float32):
    """The decoder step's types (t = 0, moving to p = -1) from the conditioned log v0_hat [n,K], the state's types vt [n] and the
    uniforms [n,K]: stepwise.step's q_v_posterior at t = 0 with the forbidden classes at -inf before the normalisation.  Returns
    (v, the normalised log posterior, Gumbel margin best minus runner-up)."""
    K = log_v0.shape[1]
    n = vt.shape[0]
    sdd = {k: sd[k].to(dtype) for k in stepwise.TABLES}
    tt = torch.zeros(1, dtype=torch.long)
    batch = torch.zeros(n, dtype=torch.long)
    with default_dtype(dtype):
        log_v = restate.index_to_log_onehot(vt, K)
        un = restate.q_v_pred(sdd, log_v0, tt, batch, K) + restate.q_v_pred_one_timestep(sdd, log_v, tt, batch, K)
        un = un.masked_fill(~allowed, float('-inf'))
        log_prob = un - torch.logsumexp(un, dim=-1, keepdim=True)
        u = v_uniform.to(dtype)
        score = -torch.log(-torch.log(u + 1e-30) + 1e-30) + log_prob
        top2 = score.topk(2, dim=-1).values
        return restate.log_sample_categorical_from_uniform(log_prob, u), log_prob, top2[:, 0] - top2[:, 1]


def conditioned_step(sd, cfg, tables, s, xt, vt, x0, logits, pos_noise, v_uniform, allowed, guide_fn=None, pos_only=False,
                     dtype=torch.float32):
    """Step s of a chain on the per-step `tables` (oracle.resample.path_tables) with the element constraint `allowed` [n,K] bool
    (None: clash_guidance.guided_jump_step itself; guide_fn as there).  Returns that function's dict: 'v0' the conditioned log v0_hat,
    and on the decoder step 'v', 'vt', 'margin' from `decoder_types`."""
    if allowed is not None:
        logits = logits.to(dtype).masked_fill(~allowed, float('-inf'))
    out = clash_guidance.guided_jump_step(sd, cfg, tables, s, xt, vt, x0, logits, pos_noise, v_uniform, guide_fn, pos_only=pos_only,
                                          dtype=dtype)
    if allowed is None or pos_only or int(tables['p'][s]) >= 0:
        return out
    assert int(tables['t'][s]) == 0
    v, log_prob, margin = decoder_types(sd, vt, out['v0'], v_uniform, allowed, dtype=dtype)
    out.update(v=v, vt=log_prob, margin=margin)
    return out


def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand, pos_noise, v_uniform,
                     time_path, center_pos_mode='protein', pos_only=False, fixed_mask=None, fixed_tape=None, start_time=None,
                     start_tape=None, allowed=None, guidance=None, step_callback=None):
    """oracle.clash_guidance.sample_diffusion with the element constraint `allowed` [Nl,K] bool at every denoising step (fixed rows
    are overwritten after the step as there).  allowed=None: that function itself.  The loop below is that function's, with
    guided_jump_step replaced by conditioned_step."""
    if allowed is None:
        return clash_guidance.sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand,
                                               pos_noise, v_uniform, time_path, center_pos_mode=center_pos_mode, pos_only=pos_only,
                                               fixed_mask=fixed_mask, fixed_tape=fixed_tape, start_time=start_time, start_tape=start_tape,
                                               guidance=guidance, step_callback=step_callback)
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    T = sd['betas'].shape[0]
    allowed = torch.as_tensor(allowed, dtype=torch.bool)
    assert tuple(allowed.shape) == (len(batch_ligand), K) and bool(allowed.any(1).all())
    tab = resample.path_tables(sd, time_path)
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, x0, offset = restate.center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        offset = torch.zeros(num_graphs, 3)
    v0 = init_ligand_v.clone()
    fm = None if fixed_mask is None else torch.as_tensor(fixed_mask, dtype=torch.bool)
    if fm is not None and not bool(fm.any()):
        fm = None
    guide_fn = None if guidance is None else (lambda y: guidance(y, protein_pos, batch_ligand, batch_protein))

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
            out = conditioned_step(sd, cfg, tab, s, ligand_pos, ligand_v, preds['pred_ligand_pos'], preds['pred_ligand_v'], pos_noise[s],
                                   v_uniform[s], allowed, guide_fn, pos_only=pos_only)
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


def sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, time_path, batch_size=16,
                            center_pos_mode='protein', sample_num_atoms='prior', fixed_ligand=None, allowed=None, guidance=None):
    """oracle.clash_guidance.sample_diffusion_ligand (the rng='cpu' driver on a time path) with the chain of `sample_diffusion` above:
    `allowed` a [K] bool set for every free atom, fragment rows every class.  allowed=None: that driver itself.  The draws are that
    driver's, in its order: the constraint draws nothing."""
    if allowed is None:
        return clash_guidance.sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, time_path,
                                                      batch_size=batch_size, center_pos_mode=center_pos_mode,
                                                      sample_num_atoms=sample_num_atoms, fixed_ligand=fixed_ligand, guidance=guidance)
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    allowed = torch.as_tensor(allowed, dtype=torch.bool)
    assert tuple(allowed.shape) == (K,)
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
        am = allowed.expand(n_lig, K).clone()
        if n_f:
            starts = np.cumsum([0] + sizes[:-1])
            rows = torch.from_numpy((starts[:, None] + np.arange(n_f)[None, :]).reshape(-1))
            mask = torch.zeros(n_lig, dtype=torch.bool)
            mask[rows] = True
            init_pos[rows] = frag_pos.repeat(n_data, 1)
            init_v = init_v.clone()
            init_v[rows] = frag_v.repeat(n_data)
            fixed = {'fixed_mask': mask, 'fixed_tape': (torch.randn(S + 1, n_lig, 3), torch.rand(S + 1, n_lig, K))}
            am[mask] = True
        r = sample_diffusion(sd, c, ppos, pfeat, batch_protein, init_pos, init_v, batch_ligand, pn, vu, time_path,
                             center_pos_mode=center_pos_mode, allowed=am, guidance=guidance, **fixed)
        cum = np.cumsum([0] + sizes)
        per = [r['pos'].numpy().astype(np.float64), r['v'].numpy(), torch.stack(r['pos_traj']).numpy().astype(np.float64),
               torch.stack(r['v_traj']).numpy(), torch.stack(r['v0_traj']).numpy(), torch.stack(r['vt_traj']).numpy()]
        for j, arr in enumerate(per):
            outs[j] += [arr[cum[k]:cum[k + 1]] if j < 2 else arr[:, cum[k]:cum[k + 1]] for k in range(n_data)]
        current_i += n_data
    return tuple(outs) + ([0.0] * num_batch,)
