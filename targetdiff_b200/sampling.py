"""sample_diffusion_ligand -- the sampling driver (reference scripts/sample_diffusion.py:31-116), same signature and
7-tuple result, running on the libtdiff engine.  Differences in mechanics, not in results: the batch of `n_data` clones
is assembled directly (no PyG Batch), trajectories come back from the device once per batch instead of 4 D2H copies per
step, and un-batching is done on stacked arrays.

Randomness.  `rng='device'` (default): initial state from torch's generator of `device`, per-step noise from the engine's
counter-based Philox stream keyed by a seed drawn from torch's CPU generator (so `seed_all` reproduces a run).
`rng='cpu'`: every draw comes from torch's global CPU generator in exactly the reference's order -- per batch
`randn_like(center)` (:63), `rand_like(uniform_logits)` (:69 via models/molopt_score_model.py:161), then per denoising step
`randn_like(ligand_pos)` and `rand_like(log_model_prob)` (models/molopt_score_model.py:678,685) -- pre-drawn as a noise tape.
A run seeded with `seed_all(s)` then consumes the same random numbers as the unmodified reference run on CPU with the same
seed, which is what "identical RNG seeds" parity needs (tests/golden/pocket_1h36_*.npz were produced that way).

Fragment-conditioned sampling (an extension beyond the reference, DESIGN.md section 1).  `fixed_ligand=(pos [n_f,3] lab frame,
v [n_f] class indices)` puts the fragment in the first n_f rows of every sample's ligand and holds those atoms to the forward process
of the fragment through the chain (ScorePosNet3D.sample_diffusion(fixed_mask=...)); they end exactly at `pos` / `v`.  Each sample's
size comes from `sample_num_atoms` as without a fragment and is raised to n_f + 1 where it is smaller, so that every sample grows at
least one atom.  The initial draws still cover every row (the fragment rows' values are replaced), so under rng='cpu' the generator
is consumed as without a fragment, followed by the fixed atoms' tape: randn(S+1, Nl, 3), then rand(S+1, Nl, K).  `pos_only=True`
keeps the reference ligand's types and cannot take a fragment.

Respaced sampling (an extension beyond the reference, DESIGN.md section 1).  `time_seq` (e.g. `respaced_time_seq(T, 100)`) runs the
chain on that decreasing subsequence of timesteps with the exact jump posteriors (ScorePosNet3D.sample_diffusion(time_seq=...)).
Under rng='cpu' the tape has S = len(time_seq) steps in the reference's interleaved order, then comes the fixed tape [S+1, ...].
Whether a checkpoint's molecules keep their quality at fewer steps has not been measured.

Start-ligand sampling (an extension beyond the reference, DESIGN.md section 1).  `start_ligand=(pos [n,3] lab frame, v [n] class
indices)` with `start_time` = t0 starts every sample from that ligand noised to t0 and runs the reverse chain from t0
(ScorePosNet3D.sample_diffusion(start_time=...)): by default t0, t0 - 1, ..., 0, or `time_seq` from t0 (e.g. respaced_time_seq(T, n,
start=t0)).  Every sample has the start ligand's n atoms (`sample_num_atoms` is not read), and no initial N(0,1) or uniform draws are
made.  `keep_atoms` (indices into the start ligand) become fixed rows, held to the forward process of their start positions and types.
Under rng='cpu' each batch draws, in this order, the start tape randn(Nl, 3), rand(Nl, K) (the uniforms skipped under pos_only), the
step tape in the reference's interleaved order, and with kept atoms the fixed tape randn(S+1, Nl, 3), rand(S+1, Nl, K) (the uniforms
skipped under pos_only).  With pos_only the types are the start ligand's.  Sample quality from a start ligand has not been measured.

Resampled sampling (an extension beyond the reference, DESIGN.md section 1; RePaint, Lugmayr et al. 2022).  `time_path` (e.g.
`resampled_time_path(base, resamplings=r, jump_length=j)`) runs a time path whose steps may go up: a re-noising step draws the whole
state back up with the forward process, so that the free atoms are denoised again next to the held fragment or kept atoms
(ScorePosNet3D.sample_diffusion(time_path=...)).  Not with `time_seq`; with a start ligand the path begins at the start time.  Under
rng='cpu' the draws are those of a time_seq of S = len(time_path) steps.  Whether resampling improves the molecules has not been
measured.

Element constraints (an extension beyond the reference, DESIGN.md section 1).  `allowed_types` restricts the classes the free atoms
end in: class indices or a [K] bool for every free atom (pocket.element_classes maps element symbols to a mode's classes), or with a
start ligand a [n, K] bool with one row per start atom (e.g. "this position must be N or O").  Fragment and kept atoms get every class.
Each denoising step conditions the type prediction on the set and the decoder step draws from the posterior renormalised over it
(ScorePosNet3D.sample_diffusion(allowed_types=...)), so a chain that ends at t = 0 uses only allowed classes; a set of every class
runs the plain chain.  No random numbers are drawn, so the rng='cpu' order is unchanged.  Not with pos_only.  Whether constrained
molecules are chemically sensible has not been measured."""
import time

import numpy as np
import torch

from . import atom_num
from .config import check_clash_guidance, check_connect_guidance
from .score_model import check_time_path, check_time_seq, log_sample_categorical


def seed_all(seed):
    """reference utils/misc.py:58-61"""
    import random
    torch.manual_seed(seed)
    np.random.seed(seed)
    random.seed(seed)


def respaced_time_seq(T, n, start=None):
    """n timesteps spaced evenly from T - 1 down to 0, each rounded to the nearest integer (half to even): a strictly decreasing
    time sequence for ScorePosNet3D.sample_diffusion(time_seq=...).  n = T gives the default chain T-1, ..., 0.  With a start time
    `start` in 0..T-1 the sequence runs from `start` down to 0 instead, with 2 <= n <= start + 1 (n = 1 when start = 0)."""
    T, n = int(T), int(n)
    if start is None:
        if not 2 <= n <= T:
            raise ValueError('respaced steps must lie in 2..T = %d, got %d' % (T, n))
        top = T - 1
    else:
        top = int(start)
        if not 0 <= top <= T - 1:
            raise ValueError('start time %d outside 0..T-1 = %d' % (top, T - 1))
        lo = 1 if top == 0 else 2
        if not lo <= n <= top + 1:
            raise ValueError('respaced steps from start time %d must lie in %d..%d, got %d' % (top, lo, top + 1, n))
    seq = [int(x) for x in np.rint(np.linspace(top, 0, n))]
    assert seq[0] == top and seq[-1] == 0 and all(b < a for a, b in zip(seq, seq[1:]))
    return seq


def resampled_time_path(base, resamplings=1, jump_length=1):
    """The RePaint time path (Lugmayr et al. 2022) over a strictly decreasing base sequence b_0 > ... > b_{n-1} >= 0 (the default chain,
    a respaced_time_seq, or one from a start time), for ScorePosNet3D.sample_diffusion(time_path=...).  The base indices fall into blocks
    [k j, e] with e = min(k j + j, n - 1); each block is denoised from b_{kj} down to b_e, then `resamplings` - 1 times re-noised in one
    step from b_e back up to b_{kj} and denoised again; the path ends with the last step at b_{n-1}.  That is r (n - 1) + 1 denoising
    and (r - 1) ceil((n - 1) / j) re-noising steps; r = 1 gives the base itself."""
    b = [int(x) for x in (base.tolist() if hasattr(base, 'tolist') else base)]
    r, j = int(resamplings), int(jump_length)
    if not b or any(y >= x for x, y in zip(b, b[1:])) or b[-1] < 0:
        raise ValueError('the base of a resampled time path must be a non-empty strictly decreasing sequence of times >= 0')
    if r < 1:
        raise ValueError('resamplings must be >= 1, got %d' % r)
    if j < 1:
        raise ValueError('jump_length must be >= 1, got %d' % j)
    n = len(b)
    path = [b[0]]
    for k0 in range(0, n - 1, j):
        e = min(k0 + j, n - 1)
        for rep in range(r):
            if rep > 0:
                path.append(b[k0])                                      # one re-noising step from b_e back up to b_{kj}
            path += b[k0 + 1:e + 1]
    return path


def _check_start(model,start_ligand, start_time, keep_atoms, fixed_ligand):
    """(pos [n,3] float32, v [n] int64, t0, keep [k] int64) of a start ligand, or None without one; ValueError for what
    sample_diffusion_ligand refuses."""
    if start_ligand is None:
        if start_time is not None or keep_atoms is not None:
            raise ValueError('start_time and keep_atoms need a start_ligand')
        return None
    if start_time is None:
        raise ValueError('a start_ligand needs a start_time')
    if fixed_ligand is not None:
        raise ValueError('fixed_ligand cannot be combined with start_ligand: keep atoms of the start ligand with keep_atoms instead')
    T = model.num_timesteps
    t0 = int(start_time)
    if not 0 <= t0 <= T - 1:
        raise ValueError('start_time %d outside 0..T-1 = %d' % (t0, T - 1))
    pos = torch.as_tensor(start_ligand[0]).detach().cpu().float()
    v = torch.as_tensor(start_ligand[1]).detach().cpu()
    n = v.shape[0] if v.dim() == 1 else -1
    if v.is_floating_point() or pos.dim() != 2 or tuple(pos.shape) != (n, 3) or n < 1:
        raise ValueError('start_ligand must be (pos [n,3], v [n] integer classes) with n >= 1; got shapes %s, %s'
                         % (tuple(pos.shape), tuple(v.shape)))
    v = v.long()
    if int(v.min()) < 0 or int(v.max()) >= model.num_classes:
        raise ValueError('start_ligand classes must lie in 0..%d' % (model.num_classes - 1))
    keep = torch.zeros(0, dtype=torch.long)
    if keep_atoms is not None:
        keep = torch.as_tensor(keep_atoms).detach().cpu().reshape(-1)
        if keep.is_floating_point():
            raise ValueError('keep_atoms must be integer indices into the start ligand')
        keep = keep.long()
        if len(keep) and (int(keep.min()) < 0 or int(keep.max()) >= n):
            raise ValueError('keep_atoms must lie in 0..%d' % (n - 1))
        if len(torch.unique(keep)) != len(keep):
            raise ValueError('keep_atoms must be unique')
        if len(keep) >= n:
            raise ValueError('keep_atoms must leave at least one of the %d start atoms free' % n)
    return pos, v, t0, keep


def _check_allowed(allowed_types, K, start, pos_only):
    """The element constraint of sample_diffusion_ligand as a [K] bool (every free atom) or [n, K] bool (each start atom), or None
    without one; ValueError for what sample_diffusion_ligand refuses."""
    if allowed_types is None:
        return None
    if pos_only:
        raise ValueError('allowed_types constrains atom types, which pos_only=True keeps as they are')
    a = torch.as_tensor(allowed_types).detach().cpu()
    if a.numel() == 0:
        raise ValueError('allowed_types is empty: every atom needs at least one allowed class')
    if a.dtype == torch.bool and a.dim() == 2:
        if start is None:
            raise ValueError('a per-atom allowed_types [n, K] needs a start_ligand: its rows are the start atoms')
        if tuple(a.shape) != (len(start[1]), K):
            raise ValueError('a per-atom allowed_types must be [n, K] = %s, got %s' % ((len(start[1]), K), tuple(a.shape)))
        m = a
    elif a.dtype == torch.bool:
        if a.dim() != 1 or len(a) != K:
            raise ValueError('a bool allowed_types must be [K] = [%d] or, with a start_ligand, [n, K]; got %s' % (K, tuple(a.shape)))
        m = a
    else:
        if a.is_floating_point() or a.is_complex() or a.dim() > 1:
            raise ValueError('allowed_types must be class indices, a [K] bool or a per-atom [n, K] bool; got %s %s' % (tuple(a.shape), a.dtype))
        idx = a.reshape(-1).long()
        if int(idx.min()) < 0 or int(idx.max()) >= K:
            raise ValueError('allowed_types classes must lie in 0..%d' % (K - 1))
        m = torch.zeros(K, dtype=torch.bool)
        m[idx] = True
    empty = (~m.reshape(-1, K).any(1)).nonzero().reshape(-1).tolist()
    if empty:
        raise ValueError('allowed_types allows no class for %s' % ('any atom' if m.dim() == 1 else 'start atom(s) %s' % empty))
    return m


def _split(arr, cum, n_data):
    return [arr[..., cum[k]:cum[k + 1], :] if arr.ndim == 3 else arr[..., cum[k]:cum[k + 1]] for k in range(n_data)]


def sample_diffusion_ligand(model, data, num_samples, batch_size=16, device='cuda:0', num_steps=None, pos_only=False,
                            center_pos_mode='protein', sample_num_atoms='prior', rng='device', fixed_ligand=None, time_seq=None,
                            start_ligand=None, start_time=None, keep_atoms=None, time_path=None, clash_radius=None, clash_strength=0.0,
                            allowed_types=None, connect_radius=None, connect_length=None, connect_strength=0.0):
    if rng not in ('device', 'cpu'):
        raise ValueError("rng must be 'device' or 'cpu'")
    clash_radius, clash_strength = check_clash_guidance(clash_radius, clash_strength)     # draws nothing: rng='cpu' order unchanged
    connect = check_connect_guidance(connect_radius, connect_length, connect_strength)    # nor does connectivity guidance
    start = _check_start(model, start_ligand, start_time, keep_atoms, fixed_ligand)
    allowed = _check_allowed(allowed_types, model.num_classes, start, pos_only)          # draws nothing either
    if time_path is not None:
        if time_seq is not None:
            raise ValueError('time_path cannot be combined with time_seq')
        time_path = check_time_path(time_path, model.num_timesteps, start=None if start is None else start[2])
        if num_steps is not None and int(num_steps) != len(time_path):
            raise ValueError('num_steps=%d disagrees with a time_path of %d steps' % (int(num_steps), len(time_path)))
    elif start is not None and time_seq is None:
        time_seq = list(range(start[2], -1, -1))
    if time_seq is not None:
        time_seq = check_time_seq(time_seq, model.num_timesteps, start=None if start is None else start[2])
        if num_steps is not None and int(num_steps) != len(time_seq):
            raise ValueError('num_steps=%d disagrees with a time_seq of %d steps' % (int(num_steps), len(time_seq)))
    n_f = 0
    if fixed_ligand is not None:
        if pos_only:
            raise ValueError('pos_only=True keeps the reference ligand\'s atom types and cannot take a fixed fragment')
        frag_pos = torch.as_tensor(fixed_ligand[0]).detach().cpu().float()
        frag_v = torch.as_tensor(fixed_ligand[1]).detach().cpu().long()
        n_f = frag_v.shape[0]
        if frag_pos.dim() != 2 or frag_pos.shape != (n_f, 3) or frag_v.dim() != 1 or n_f < 1:
            raise ValueError('fixed_ligand must be (pos [n_f,3], v [n_f]) with n_f >= 1; got shapes %s, %s'
                             % (tuple(frag_pos.shape), tuple(frag_v.shape)))
        if int(frag_v.min()) < 0 or int(frag_v.max()) >= model.num_classes:
            raise ValueError('fixed_ligand classes must lie in 0..%d' % (model.num_classes - 1))
    all_pred_pos, all_pred_v = [], []
    all_pred_pos_traj, all_pred_v_traj = [], []
    all_pred_v0_traj, all_pred_vt_traj = [], []
    time_list = []
    num_batch = int(np.ceil(num_samples / batch_size))
    current_i = 0
    device = torch.device(device)
    protein_pos_cpu = data.protein_pos.detach().cpu().float()
    n_prot = protein_pos_cpu.shape[0]
    protein_pos_dev = protein_pos_cpu.to(device)
    protein_feat_dev = data.protein_atom_feature.detach().to(device).float()
    for i in range(num_batch):
        n_data = batch_size if i < num_batch - 1 else num_samples - batch_size * (num_batch - 1)
        t1 = time.time()
        with torch.no_grad():
            batch_protein = torch.repeat_interleave(torch.arange(n_data, device=device), n_prot)
            if start is not None:                                       # every sample is the start ligand
                ligand_num_atoms = [len(start[1])] * n_data
            elif sample_num_atoms == 'prior':
                pocket_size = atom_num.get_space_size(protein_pos_cpu.numpy())
                ligand_num_atoms = [int(atom_num.sample_atom_num(pocket_size)) for _ in range(n_data)]
            elif sample_num_atoms == 'range':
                ligand_num_atoms = list(range(current_i + 1, current_i + n_data + 1))
            elif sample_num_atoms == 'ref':
                ligand_num_atoms = [int(data.ligand_element.size(0))] * n_data
            else:
                raise ValueError
            if n_f:
                ligand_num_atoms = [max(n, n_f + 1) for n in ligand_num_atoms]
            batch_ligand = torch.repeat_interleave(torch.arange(n_data), torch.tensor(ligand_num_atoms)).to(device)
            protein_pos = protein_pos_dev.repeat(n_data, 1)
            protein_v = protein_feat_dev.repeat(n_data, 1)

            # init ligand pos: pocket centre + N(0, 1)   (reference :61-63; scatter_mean = sequential sum / count, every clone
            # of the pocket has the same centre)
            n_lig = len(batch_ligand)
            extra = {} if time_seq is None else {'time_seq': time_seq}
            if time_path is not None:
                extra['time_path'] = time_path
            if clash_strength > 0:                                      # off is sample_diffusion's default
                extra.update(clash_radius=clash_radius, clash_strength=clash_strength)
            if connect[2] > 0:
                extra.update(connect_radius=connect[0], connect_length=connect[1], connect_strength=connect[2])
            if start is not None:                                       # the clean start ligand; the engine noises it to t0
                init_ligand_pos = start[0].to(device).repeat(n_data, 1)
                init_ligand_v = start[1].to(device).repeat(n_data)
                extra['start_time'] = start[2]
                if rng == 'cpu':
                    extra['start_noise_tape'] = (torch.randn(n_lig, 3), None if pos_only else torch.rand(n_lig, model.num_classes))
            else:
                center = (torch.zeros(1, 3).index_add_(0, torch.zeros(n_prot, dtype=torch.long), protein_pos_cpu) / max(n_prot, 1)).to(device)
                draw_dev = device if rng == 'device' else 'cpu'
                init_ligand_pos = center.expand(n_lig, 3) + torch.randn(n_lig, 3, device=draw_dev).to(device)
                # init ligand v (reference :66-70)
                if pos_only:
                    init_ligand_v = data.ligand_atom_feature_full.to(device).repeat(n_data)
                else:
                    uniform_logits = torch.zeros(n_lig, model.num_classes, device=draw_dev)
                    init_ligand_v = log_sample_categorical(uniform_logits).to(device)
            tape = None
            if rng == 'cpu':
                S = len(time_seq) if time_seq is not None else len(time_path) if time_path is not None else \
                    model.num_timesteps if num_steps is None else int(num_steps)
                pn = torch.empty(S, n_lig, 3)
                vu = torch.zeros(S, n_lig, model.num_classes)
                for st in range(S):                                     # the reference's interleaved draw order
                    pn[st] = torch.randn(n_lig, 3)
                    if not pos_only:
                        vu[st] = torch.rand(n_lig, model.num_classes)
                tape = (pn, vu)
            if start is not None and len(start[3]):
                starts = np.cumsum([0] + ligand_num_atoms[:-1])
                rows = torch.from_numpy((starts[:, None] + start[3].numpy()[None, :]).reshape(-1)).to(device)
                mask = torch.zeros(n_lig, dtype=torch.bool, device=device)
                mask[rows] = True
                extra['fixed_mask'] = mask
                if rng == 'cpu':
                    extra['fixed_noise_tape'] = (torch.randn(S + 1, n_lig, 3),
                                                 None if pos_only else torch.rand(S + 1, n_lig, model.num_classes))
            if n_f:
                starts = np.cumsum([0] + ligand_num_atoms[:-1])
                rows = torch.from_numpy((starts[:, None] + np.arange(n_f)[None, :]).reshape(-1)).to(device)
                mask = torch.zeros(n_lig, dtype=torch.bool, device=device)
                mask[rows] = True
                init_ligand_pos[rows] = frag_pos.to(device).repeat(n_data, 1)
                init_ligand_v = init_ligand_v.clone()
                init_ligand_v[rows] = frag_v.to(device).repeat(n_data)
                extra['fixed_mask'] = mask
                if rng == 'cpu':
                    extra['fixed_noise_tape'] = (torch.randn(S + 1, n_lig, 3), torch.rand(S + 1, n_lig, model.num_classes))
            if allowed is not None:                                     # fragment and kept rows: every class
                am = allowed.expand(n_lig, -1).clone() if allowed.dim() == 1 else allowed.repeat(n_data, 1)
                am = am.to(device)
                if 'fixed_mask' in extra:
                    am[extra['fixed_mask']] = True
                if not bool(am.all()):
                    extra['allowed_types'] = am

            r = model.sample_diffusion(protein_pos=protein_pos, protein_v=protein_v, batch_protein=batch_protein,
                                       init_ligand_pos=init_ligand_pos, init_ligand_v=init_ligand_v, batch_ligand=batch_ligand,
                                       num_steps=num_steps, pos_only=pos_only, center_pos_mode=center_pos_mode, stack_traj=True,
                                       noise_tape=tape, **extra)
            cum = np.cumsum([0] + ligand_num_atoms)
            pos = r['pos'].cpu().numpy().astype(np.float64)
            all_pred_pos += [pos[cum[k]:cum[k + 1]] for k in range(n_data)]
            pos_traj = r['pos_traj'].numpy().astype(np.float64)                   # [S, Nl, 3]
            all_pred_pos_traj += _split(pos_traj, cum, n_data)                    # n_data * [S, n_k, 3]
            v = r['v'].cpu().numpy()
            all_pred_v += [v[cum[k]:cum[k + 1]] for k in range(n_data)]
            all_pred_v_traj += _split(r['v_traj'].numpy(), cum, n_data)
            if not pos_only:
                all_pred_v0_traj += _split(r['v0_traj'].numpy(), cum, n_data)
                all_pred_vt_traj += _split(r['vt_traj'].numpy(), cum, n_data)
        t2 = time.time()
        time_list.append(t2 - t1)
        current_i += n_data
    return all_pred_pos, all_pred_v, all_pred_pos_traj, all_pred_v_traj, all_pred_v0_traj, all_pred_vt_traj, time_list
