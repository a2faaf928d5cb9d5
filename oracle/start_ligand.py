"""Start-ligand sampling restated on the CPU (TEST INFRASTRUCTURE, torch-CPU fp32; float64 Python for the Philox stream).

An extension beyond the reference (DESIGN.md section 1): the reverse chain starts from a given ligand (x0, v0) noised to a start time
t0 with the forward process and runs from t0 to 0.  Before the first step every row that is not fixed becomes a sample of
q(x_t0 | x0), q(v_t0 | v0) (`oracle.fixed_atoms.forward_sample`: the reference's position perturbation, models/molopt_score_model.py:
500-504, and q_v_sample, :394-398); fixed (kept) rows get their fixed-atom draw 0 at t0 instead of T - 1.  The chain is then the
respaced chain from tau_0 = t0 (`oracle.respaced`), each step `respaced.jump_step` on `restate.forward`'s outputs.

The engine's start stream uses the sampler's Philox key, counter layout and transforms (oracle/philox.py) on two more domain words:
atom a, position counter (a, 0, 0, 'stps'), class c from word c % 4 of (a, 0, 1 + c // 4, 'sttv').
"""
import numpy as np
import torch

from . import fixed_atoms, philox, respaced, restate
from .synth import DEFAULT_MODEL_CONFIG

START_POS_DOMAIN, START_TYPE_DOMAIN = 0x73747073, 0x73747476


# ----------------------------------------------------------------------------------------------------------------- noise
def start_position_normals(seed, atoms):
    """float64 normals [..., 3] of the start stream for an integer array `atoms`."""
    k0, k1 = philox.split_key(seed)
    x, y, z, w = philox.philox4x32_10(atoms, 0, 0, START_POS_DOMAIN, k0, k1)
    u0, u1, u2, u3 = 1.0 - philox.u01(x), philox.u01(y), 1.0 - philox.u01(z), philox.u01(w)
    ra, rb = np.sqrt(-2.0 * np.log(u0)), np.sqrt(-2.0 * np.log(u2))
    return np.stack([ra * np.cos(2 * np.pi * u1), ra * np.sin(2 * np.pi * u1), rb * np.cos(2 * np.pi * u3)], -1)


def start_type_uniforms(seed, atoms, K):
    """float64 uniforms [..., K] of the start stream for an integer array `atoms`."""
    k0, k1 = philox.split_key(seed)
    lanes = []
    for blk in range((K + 3) // 4):
        lanes += philox.philox4x32_10(atoms, 0, 1 + blk, START_TYPE_DOMAIN, k0, k1)
    return np.stack([philox.u01(w) for w in lanes[:K]], -1)


def start_tape(seed, n_lig, K, pos_only=False):
    """The start draw the engine makes for `seed`, as the start tape (pos_noise [Nl, 3], v_uniform [Nl, K]) of
    ScorePosNet3D.sample_diffusion(start_noise_tape=...).  Every atom has its draw; the engine reads those of the free rows only.
    With `pos_only` the uniforms are zeros, as in philox.engine_tape."""
    a = np.arange(n_lig, dtype=np.uint32)
    pn = start_position_normals(seed, a).astype(np.float32).reshape(n_lig, 3)
    if pos_only:
        vu = np.zeros((n_lig, K), np.float32)
    else:
        vu = start_type_uniforms(seed, a, K).astype(np.float32).reshape(n_lig, K)
    return torch.from_numpy(pn), torch.from_numpy(vu)


# ----------------------------------------------------------------------------------------------------------------- chain
def start_state(sd, x0, v0, batch, t0, start_tape, K, pos_only=False, fixed_mask=None, fixed_tape=None):
    """The state before the first step of a chain from the start ligand (x0 [Nl,3] centred, v0 [Nl]) at t0: the free rows a sample of
    q(x_t0 | x0), q(v_t0 | v0) from `start_tape` = (pos_noise [Nl,3], v_uniform [Nl,K] or None), the rows of `fixed_mask` their draw
    0 of `fixed_tape` = (pos_noise [S+1,Nl,3], v_uniform [S+1,Nl,K] or None) at t0."""
    n = x0.shape[0]
    fm = torch.zeros(n, dtype=torch.bool) if fixed_mask is None else torch.as_tensor(fixed_mask, dtype=torch.bool)
    pos, v = x0.clone(), v0.clone()
    draws = [(~fm, start_tape[0], start_tape[1])]
    if bool(fm.any()):
        draws.append((fm, fixed_tape[0][0], None if fixed_tape[1] is None else fixed_tape[1][0]))
    for rows, pn, vu in draws:
        vu = torch.zeros(n, K) if vu is None else vu
        pos[rows], v[rows] = fixed_atoms.forward_sample(sd, x0[rows], v0[rows], batch[rows], t0, pn[rows], vu[rows], K, pos_only)
    return pos, v


def sample_diffusion(sd, cfg, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand, pos_noise, v_uniform,
                     start_time, start_tape, time_seq=None, center_pos_mode='protein', pos_only=False, fixed_mask=None, fixed_tape=None,
                     step_callback=None):
    """The chain from the start ligand (init_ligand_pos lab frame, init_ligand_v) at `start_time` = t0 on the noise tape
    pos_noise [S,Nl,3], v_uniform [S,Nl,K], the start tape (pos_noise [Nl,3], v_uniform [Nl,K] or None) and, with `fixed_mask`, the
    fixed tape (pos_noise [S+1,Nl,3], v_uniform [S+1,Nl,K] or None): `start_state`, then the steps of `time_seq` (default t0, ..., 0),
    step s at t = tau_s moving the state to p (respaced.targets) with the fixed rows resampled at p from fixed tape row s + 1 (x0, v0
    themselves when p < 0).  Returns the reference's dict, trajectories as lists; entry s is the state after step s."""
    cfg = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    t0 = int(start_time)
    seq = list(range(t0, -1, -1)) if time_seq is None else [int(x) for x in time_seq]
    assert seq[0] == t0, 'the time sequence must begin at the start time'
    tab = respaced.jump_tables(sd, seq)
    num_graphs = int(batch_protein.max()) + 1
    protein_pos, x0, offset = restate.center_pos(protein_pos, init_ligand_pos, batch_protein, batch_ligand, center_pos_mode)
    if not torch.is_tensor(offset):
        offset = torch.zeros(num_graphs, 3)
    v0 = init_ligand_v.clone()
    fm = None if fixed_mask is None else torch.as_tensor(fixed_mask, dtype=torch.bool)
    ligand_pos, ligand_v = start_state(sd, x0, v0, batch_ligand, t0, start_tape, K, pos_only, fm, fixed_tape)
    pos_traj, v_traj, v0_traj, vt_traj = [], [], [], []
    for s, (t, p) in enumerate(zip(tab['t'].tolist(), tab['p'].tolist())):
        tt = torch.full((num_graphs,), t, dtype=torch.long)
        preds = restate.forward(sd, cfg, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step=tt)
        out = respaced.jump_step(sd, cfg, tab, s, ligand_pos, ligand_v, preds['pred_ligand_pos'], preds['pred_ligand_v'], pos_noise[s],
                                 v_uniform[s], pos_only=pos_only)
        ligand_pos, ligand_v = out['pos'], out['v']
        if not pos_only:
            v0_traj.append(out['v0'].clone()); vt_traj.append(out['vt'].clone())
        if fm is not None and bool(fm.any()):
            vu = torch.zeros(len(batch_ligand), K) if fixed_tape[1] is None else fixed_tape[1][s + 1]
            ligand_pos, ligand_v = ligand_pos.clone(), ligand_v.clone()
            ligand_pos[fm], ligand_v[fm] = fixed_atoms.forward_sample(sd, x0[fm], v0[fm], batch_ligand[fm], p, fixed_tape[0][s + 1][fm],
                                                                      vu[fm], K, pos_only)
        pos_traj.append((ligand_pos + offset[batch_ligand]).clone())
        v_traj.append(ligand_v.clone())
        if step_callback is not None:
            step_callback(s, t, preds, ligand_pos, ligand_v)
    return {'pos': ligand_pos + offset[batch_ligand], 'v': ligand_v, 'pos_traj': pos_traj, 'v_traj': v_traj,
            'v0_traj': v0_traj, 'vt_traj': vt_traj}


# ----------------------------------------------------------------------------------------------------------------- driver
def sample_diffusion_ligand(sd, cfg, protein_pos, protein_atom_feature, num_samples, start_ligand, start_time, time_seq=None,
                            keep_atoms=None, batch_size=16, center_pos_mode='protein', pos_only=False):
    """The rng='cpu' driver (targetdiff_b200.sampling.sample_diffusion_ligand) with a start ligand (pos [n,3] lab frame, v [n]) shared
    by every sample: no size draws and no initial draws; per batch the start tape randn(Nl, 3), rand(Nl, K), then S steps of
    randn(Nl, 3) / rand(Nl, K) interleaved, then with `keep_atoms` the fixed tape randn(S+1, Nl, 3), rand(S+1, Nl, K); every rand is
    skipped under pos_only.  Returns the reference's 7-tuple; the time list holds zeros."""
    c = dict(DEFAULT_MODEL_CONFIG, **(cfg or {}))
    K = sd['v_inference.2.weight'].shape[0]
    t0 = int(start_time)
    seq = list(range(t0, -1, -1)) if time_seq is None else [int(x) for x in time_seq]
    S = len(seq)
    pos0, v0 = torch.as_tensor(start_ligand[0]).float(), torch.as_tensor(start_ligand[1]).long()
    n = len(v0)
    keep = None if keep_atoms is None else torch.as_tensor(keep_atoms).long().reshape(-1)
    all_pos, all_v, all_pos_traj, all_v_traj, all_v0_traj, all_vt_traj, time_list = [], [], [], [], [], [], []
    num_batch = int(np.ceil(num_samples / batch_size))
    n_prot = protein_pos.shape[0]
    for i in range(num_batch):
        n_data = batch_size if i < num_batch - 1 else num_samples - batch_size * (num_batch - 1)
        batch_protein = torch.repeat_interleave(torch.arange(n_data), n_prot)
        ppos = protein_pos.float().repeat(n_data, 1)
        pfeat = protein_atom_feature.float().repeat(n_data, 1)
        batch_ligand = torch.repeat_interleave(torch.arange(n_data), n)
        n_lig = len(batch_ligand)
        st = (torch.randn(n_lig, 3), None if pos_only else torch.rand(n_lig, K))
        pn = torch.empty(S, n_lig, 3)
        vu = torch.zeros(S, n_lig, K)
        for s in range(S):
            pn[s] = torch.randn(n_lig, 3)
            if not pos_only:
                vu[s] = torch.rand(n_lig, K)
        fixed = {}
        if keep is not None and len(keep):
            mask = torch.zeros(n_lig, dtype=torch.bool)
            mask[(torch.arange(n_data)[:, None] * n + keep[None, :]).reshape(-1)] = True
            fixed = {'fixed_mask': mask, 'fixed_tape': (torch.randn(S + 1, n_lig, 3), None if pos_only else torch.rand(S + 1, n_lig, K))}
        r = sample_diffusion(sd, c, ppos, pfeat, batch_protein, pos0.repeat(n_data, 1), v0.repeat(n_data), batch_ligand, pn, vu, t0, st,
                             seq, center_pos_mode=center_pos_mode, pos_only=pos_only, **fixed)
        pos = r['pos'].numpy().astype(np.float64)
        all_pos += [pos[k * n:(k + 1) * n] for k in range(n_data)]
        ptraj = torch.stack(r['pos_traj']).numpy().astype(np.float64)
        all_pos_traj += [ptraj[:, k * n:(k + 1) * n] for k in range(n_data)]
        v = r['v'].numpy()
        all_v += [v[k * n:(k + 1) * n] for k in range(n_data)]
        vtraj = torch.stack(r['v_traj']).numpy()
        all_v_traj += [vtraj[:, k * n:(k + 1) * n] for k in range(n_data)]
        if not pos_only:
            v0t, vtt = torch.stack(r['v0_traj']).numpy(), torch.stack(r['vt_traj']).numpy()
            all_v0_traj += [v0t[:, k * n:(k + 1) * n] for k in range(n_data)]
            all_vt_traj += [vtt[:, k * n:(k + 1) * n] for k in range(n_data)]
        time_list.append(0.0)
    return all_pos, all_v, all_pos_traj, all_v_traj, all_v0_traj, all_vt_traj, time_list
