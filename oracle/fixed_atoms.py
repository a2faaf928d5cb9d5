"""Fixed atoms (fragment-conditioned sampling) restated on the CPU (TEST INFRASTRUCTURE, torch-CPU fp32).

An extension beyond the reference (DESIGN.md section 1): ligand atoms marked fixed are held to the forward process of a target
(x0_f, v0_f) through the reverse chain.  Everything here is made of `oracle.restate`'s pinned pieces -- the forward network, the
posteriors, the schedules -- plus the reference's own forward process (the position perturbation, models/molopt_score_model.py:500-504,
and q_v_sample, :394-398).  `sample_diffusion` with no fixed set is `restate.sample_diffusion` bit for bit (tests/test_fixed_atoms.py).

The engine's fixed-atom stream (`fixed_tape`) uses the sampler's Philox key, counter layout and transforms (oracle/philox.py) on two
more domain words: draw d of atom a, position counter (a, d, 0, 'fxps'), class c from word c % 4 of (a, d, 1 + c // 4, 'fxtv');
d = 0 before the first step, d = j + 1 after step j.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import philox, restate
from .synth import DEFAULT_MODEL_CONFIG

FIX_POS_DOMAIN, FIX_TYPE_DOMAIN = 0x66787073, 0x66787476


# ----------------------------------------------------------------------------------------------------------------- noise
def fixed_position_normals(seed, atoms, draws):
    """float64 normals [..., 3] of the fixed-atom stream for broadcastable integer arrays `atoms`, `draws`."""
    k0, k1 = philox.split_key(seed)
    x, y, z, w = philox.philox4x32_10(atoms, draws, 0, FIX_POS_DOMAIN, k0, k1)
    u0, u1, u2, u3 = 1.0 - philox.u01(x), philox.u01(y), 1.0 - philox.u01(z), philox.u01(w)
    ra, rb = np.sqrt(-2.0 * np.log(u0)), np.sqrt(-2.0 * np.log(u2))
    return np.stack([ra * np.cos(2 * np.pi * u1), ra * np.sin(2 * np.pi * u1), rb * np.cos(2 * np.pi * u3)], -1)


def fixed_type_uniforms(seed, atoms, draws, K):
    """float64 uniforms [..., K] of the fixed-atom stream for broadcastable integer arrays `atoms`, `draws`."""
    k0, k1 = philox.split_key(seed)
    lanes = []
    for blk in range((K + 3) // 4):
        lanes += philox.philox4x32_10(atoms, draws, 1 + blk, FIX_TYPE_DOMAIN, k0, k1)
    return np.stack([philox.u01(w) for w in lanes[:K]], -1)


def fixed_tape(seed, n_lig, num_steps, K, pos_only=False):
    """The fixed atoms' draws the engine makes for `seed` over a chain of `num_steps` steps, as the fixed-atom tape
    (pos_noise [S+1, Nl, 3], v_uniform [S+1, Nl, K]) of ScorePosNet3D.sample_diffusion(fixed_noise_tape=...).  Every atom has its
    draws; the engine reads those of the fixed rows only.  With `pos_only` the uniforms are zeros, as in philox.engine_tape."""
    d = np.arange(num_steps + 1, dtype=np.uint32)[:, None]
    a = np.arange(n_lig, dtype=np.uint32)[None, :]
    pn = fixed_position_normals(seed, a, d).astype(np.float32)
    if pos_only:
        vu = np.zeros((num_steps + 1, n_lig, K), np.float32)
    else:
        vu = fixed_type_uniforms(seed, a, d, K).astype(np.float32)
    return torch.from_numpy(pn), torch.from_numpy(vu)


# ----------------------------------------------------------------------------------------------------------------- chain
def forward_sample(sd, x0, v0, batch, tm, eps, uniform, K, pos_only=False):
    """A sample of q(x_tm | x0), q(v_tm | v0) from normals `eps` [n,3] and uniforms `uniform` [n,K] -- the position perturbation
    sqrt(ac) x0 + sqrt(1 - ac) eps (:500-504) and Gumbel-max over the unnormalised q_v_pred(log_onehot(v0), tm) (:394-398) -- or x0
    and v0 themselves when tm < 0.  With `pos_only` the types are returned unchanged."""
    if tm < 0:
        return x0.clone(), v0.clone()
    a = sd['alphas_cumprod'][tm]
    x = a.sqrt() * x0 + (1.0 - a).sqrt() * eps
    if pos_only:
        return x, v0.clone()
    t = torch.full((int(batch.max()) + 1 if len(batch) else 1,), tm, dtype=torch.long)
    log_q = restate.q_v_pred(sd, restate.index_to_log_onehot(v0, K), t, batch, K)
    return x, restate.log_sample_categorical_from_uniform(log_q, uniform)


def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand,
                     pos_noise, v_uniform, fixed_mask, fixed_tape, num_steps=None, center_pos_mode='protein', step_callback=None,
                     pos_only=False):
    """restate.sample_diffusion with the rows `fixed_mask` [Nl] bool held to the forward process of their initial rows (x0_f, v0_f),
    on the fixed-atom tape `fixed_tape` = (pos_noise [S+1,Nl,3], v_uniform [S+1,Nl,K]):
      before the first step they become a sample of q(x_{T-1} | x0_f), q(v_{T-1} | v0_f) from tape row 0;
      after the step at time t (network and posterior update unchanged for every row) a fresh sample at t - 1 from tape row s + 1,
      or x0_f, v0_f themselves after t = 0.
    pos_traj / v_traj record the overwritten state, v0_traj / vt_traj the model's.  The loop is restate.sample_diffusion's
    (models/molopt_score_model.py:633-703) with the overwrite added."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    assert cfg['model_mean_type'] in ('C0', 'noise')
    T = sd['betas'].shape[0]
    K = sd['v_inference.2.weight'].shape[0]
    if num_steps is None:
        num_steps = T
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, ligand_pos, offset = restate.center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        offset = torch.zeros(num_graphs, 3)
    ligand_v = init_ligand_v
    fm = torch.as_tensor(fixed_mask, dtype=torch.bool)
    assert fm.shape == (len(batch_ligand),), 'fixed_mask must have one entry per ligand atom'
    fpn, fvu = fixed_tape
    x0f, v0f, bf = ligand_pos[fm].clone(), ligand_v[fm].clone(), batch_ligand[fm]

    def hold(pos, v, d, tm):
        pos, v = pos.clone(), v.clone()
        pos[fm], v[fm] = forward_sample(sd, x0f, v0f, bf, tm, fpn[d][fm], fvu[d][fm], K, pos_only)
        return pos, v

    ligand_pos, ligand_v = hold(ligand_pos, ligand_v, 0, T - 1)
    pos_traj, v_traj, v0_traj, vt_traj = [], [], [], []
    time_seq = list(reversed(range(T - num_steps, T)))
    for s, i in enumerate(time_seq):
        t = torch.full((num_graphs,), i, dtype=torch.long)
        preds = restate.forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step=t)
        pos0, v0 = preds['pred_ligand_pos'], preds['pred_ligand_v']
        if cfg['model_mean_type'] == 'noise':
            eps = pos0 - ligand_pos
            pos0 = restate.extract(sd['sqrt_recip_alphas_cumprod'], t, batch_ligand) * ligand_pos - \
                restate.extract(sd['sqrt_recipm1_alphas_cumprod'], t, batch_ligand) * eps
        pos_mean = restate.q_pos_posterior(sd, pos0, ligand_pos, t, batch_ligand)
        logvar = restate.extract(sd['posterior_logvar'], t, batch_ligand)
        nonzero = (1 - (t == 0).float())[batch_ligand].unsqueeze(-1)
        ligand_pos = pos_mean + nonzero * (0.5 * logvar).exp() * pos_noise[s]
        if not pos_only:
            log_v_recon = F.log_softmax(v0, dim=-1)
            log_v = restate.index_to_log_onehot(ligand_v, K)
            log_model_prob = restate.q_v_posterior(sd, log_v_recon, log_v, t, batch_ligand, K)
            ligand_v = restate.log_sample_categorical_from_uniform(log_model_prob, v_uniform[s])
            v0_traj.append(log_v_recon.clone()); vt_traj.append(log_model_prob.clone())
        ligand_pos, ligand_v = hold(ligand_pos, ligand_v, s + 1, i - 1)          # the overwrite, after the step
        pos_traj.append((ligand_pos + offset[batch_ligand]).clone())
        v_traj.append(ligand_v.clone())
        if step_callback is not None:
            step_callback(s, i, preds, ligand_pos, ligand_v)
    return {'pos': ligand_pos + offset[batch_ligand], 'v': ligand_v, 'pos_traj': pos_traj, 'v_traj': v_traj,
            'v0_traj': v0_traj, 'vt_traj': vt_traj}


# ----------------------------------------------------------------------------------------------------------------- driver
def sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, prior, fixed_ligand, batch_size=16,
                            num_steps=None, center_pos_mode='protein', sample_num_atoms='prior'):
    """restate.sample_diffusion_ligand (scripts/sample_diffusion.py:31-116 on the global CPU generators) with a fragment
    `fixed_ligand` = (pos [n_f,3] lab frame, v [n_f]): it occupies the first n_f rows of every sample, sizes below n_f + 1 are raised to
    n_f + 1, the initial draws still cover every row (the fragment rows' values are replaced), and after the batch's draws come the fixed
    tape's randn(S+1, Nl, 3), then rand(S+1, Nl, K).  Not with pos_only (the reference ligand's types)."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    T = sd['betas'].shape[0]
    S = T if num_steps is None else num_steps
    frag_pos = torch.as_tensor(fixed_ligand[0]).float()
    frag_v = torch.as_tensor(fixed_ligand[1]).long()
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
        starts = np.cumsum([0] + sizes[:-1])
        rows = torch.from_numpy((starts[:, None] + np.arange(n_f)[None, :]).reshape(-1))
        mask = torch.zeros(n_lig, dtype=torch.bool)
        mask[rows] = True
        init_pos[rows] = frag_pos.repeat(n_data, 1)
        init_v = init_v.clone()
        init_v[rows] = frag_v.repeat(n_data)
        ft = (torch.randn(S + 1, n_lig, 3), torch.rand(S + 1, n_lig, K))
        r = sample_diffusion(sd, c, ppos, pfeat, batch_protein, init_pos, init_v, batch_ligand, pn, vu, mask, ft, num_steps=num_steps,
                             center_pos_mode=center_pos_mode)
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
