"""Command line for the sampling path (same arguments / outputs as the reference's scripts).

    python -m targetdiff_b200.cli sample_for_pocket configs/sampling.yml --pdb_path pocket.pdb [--num_samples N] [--result_path DIR]
            [--fragment FILE | --start_ligand FILE]
        (reference scripts/sample_for_pocket.py:34-93: sample ligands into one pocket given as a PDB file; --fragment FILE, a .pt or
        .npz holding 'pos' [n,3] (the PDB's frame) and 'v' [n] class indices, grows every sample from that fragment: its atoms are
        the first n of each ligand and end exactly at 'pos' / 'v', see targetdiff_b200.sampling.  sample.pt then also holds
        'fixed_ligand_atoms': n.  --start_ligand FILE, the same kind of file with an optional integer 'keep' [k] of atom indices,
        starts every sample from that ligand noised to `sample.start_time` (required in the config with it) and keeps the 'keep'
        atoms; sample.pt then also holds 'start_ligand' (pos, v), 'start_time', 'kept_atoms' and, with sample.respaced_steps,
        'time_seq')

    [torchrun --nproc-per-node N -m] python -m targetdiff_b200.cli sample_pockets configs/sampling.yml --pocket_dir DIR | --pocket_list FILE
            [-i ID] [--schedule round_robin|longest_first] [--result_path DIR] [--num_samples N] [--batch_size B]
        (reference scripts/sample_diffusion.py:118-186 + scripts/batch_sample_diffusion.sh: pocket i -> `result_{i}.pt`, pockets
        assigned to workers round-robin; here the workers are the ranks of one torchrun job, one weight broadcast, no other collective)

    python -m targetdiff_b200.cli score_ligands configs/sampling.yml (--pdb_path P --ligand FILE [FILE ...] | --samples RESULT.pt)
            [--time_steps N|all] [--batch_size B] [--embedding] [--result_path DIR] [--device D]
        (reference scripts/likelihood_est_diffusion.py: the variational-bound NLL of each ligand, targetdiff_b200.likelihood.ligand_nll;
        --ligand files as --fragment's, in the --pdb_path pocket; --samples scores every molecule of a sample.pt / result_{i}.pt in its
        own 'data' pocket.  Seeded by sample.seed.  Writes <result_path>/scores.pt: one dict per ligand in input order with 'kl_pos',
        'kl_v' [n_t + 1] (the last entry the prior), 'nll', with --embedding 'pred_ligand_v', 'final_h', 'final_ligand_h', and
        'source' (plus 'sample_index' with --samples))

Result file: `<result_path>/sample.pt` (sample_for_pocket) or `<result_path>/result_{i}.pt` (sample_pockets) = {'data', 'pred_ligand_pos', 'pred_ligand_v', 'pred_ligand_pos_traj', 'pred_ligand_v_traj', 'time'}
-- the schema scripts/sample_diffusion.py:175-182 writes and scripts/evaluate_diffusion.py:70-76 reads (positions float64, per-sample
lists; trajectories [steps, atoms, 3]).  With `sample.respaced_steps: n` in the config (an extension beyond the reference) both commands
run the n-step chain of sampling.respaced_time_seq(T, n) instead of num_steps, and the result also holds 'time_seq'.  With
`sample.resamplings: r` > 1 (and `sample.jump_length: j`, default 1) sample_for_pocket runs sampling.resampled_time_path over that
chain, with a --fragment or kept atoms only, and sample.pt also holds 'time_path'; sample_pockets refuses the key.  With
`sample.clash_strength: lambda` > 0 and `sample.clash_radius: rho` (config.sample_clash_guidance; strength 0, the default, is off) both
commands run clash guidance (ScorePosNet3D.sample_diffusion), and the result also holds 'clash_guidance': {'radius', 'strength'}.  With
`sample.allowed_elements: [C, N, O, ...]` or `sample.allowed_classes: [...]` (config.sample_allowed_classes, in the checkpoint's
ligand_atom_mode) both commands constrain every free atom of the finished molecules to those classes, and the result also holds
'allowed_classes'.  With `sample.connect_strength: lambda` > 0, `sample.connect_radius: rho` and `sample.connect_length: b`
(config.sample_connect_guidance; strength 0, the default, is off) both commands run connectivity guidance, and the result also holds
'connect_guidance': {'radius', 'length', 'strength'}.  Molecule
reconstruction / SDF writing needs RDKit + OpenBabel and stays out of scope."""
import argparse
import os
import shutil
import sys

import torch

from .config import (check_resampling, load_config, sample_allowed_classes, sample_clash_guidance, sample_connect_guidance, sampling_start,
                     sampling_time_path, sampling_time_seq)
from .likelihood import likelihood_time_steps, ligand_nll
from .pocket import LIGAND_CLASS_ELEMENTS, pdb_to_pocket_data
from .sampling import sample_diffusion_ligand, seed_all
from .score_model import ScorePosNet3D


PROTEIN_FEATURE_DIM = 27                                                    # reference utils/transforms.py:115-132
LIGAND_ATOM_MODE_CLASSES = {m: len(z) for m, z in LIGAND_CLASS_ELEMENTS.items()}   # len(MAP_ATOM_TYPE_*_TO_INDEX), utils/transforms.py:11-66,143-149


def build_result(data, outputs):
    pred_pos, pred_v, pred_pos_traj, pred_v_traj, pred_v0_traj, pred_vt_traj, time_list = outputs
    return {'data': data, 'pred_ligand_pos': pred_pos, 'pred_ligand_v': pred_v, 'pred_ligand_pos_traj': pred_pos_traj,
            'pred_ligand_v_traj': pred_v_traj, 'time': time_list}


def _allowed_classes(config, model):
    """The element constraint of the config (config.sample_allowed_classes) in the checkpoint's ligand atom mode, or None."""
    if config.sample.get('allowed_elements') is None and config.sample.get('allowed_classes') is None:
        return None
    return sample_allowed_classes(config.sample, model.ligand_atom_mode)


def add_allowed_classes(result, allowed):
    """Record an element constraint in a result dict; nothing without one, so the file is as without it."""
    if allowed is not None:
        result['allowed_classes'] = list(allowed)
    return result


def add_clash_guidance(result, radius, strength):
    """Record a clash-guidance setting in a result dict; nothing when guidance is off, so the file is as without it."""
    if strength > 0:
        result['clash_guidance'] = {'radius': radius, 'strength': strength}
    return result


def add_connect_guidance(result, radius, length, strength):
    """Record a connectivity-guidance setting in a result dict; nothing when guidance is off, so the file is as without it."""
    if strength > 0:
        result['connect_guidance'] = {'radius': radius, 'length': length, 'strength': strength}
    return result


def _load_model(config, device, rank=0):
    """Checkpoint -> engine-backed model on `device`.  Under torchrun only rank 0's weights count: one flat broadcast
    (targetdiff_b200.dist.broadcast_state_dict) replaces the per-process checkpoint parsing of the reference's shell loop."""
    from . import dist as tdist
    ckpt = torch.load(config.model.checkpoint, map_location='cpu', weights_only=False)
    tc = ckpt['config']
    get = (lambda c, k: getattr(c, k)) if hasattr(tc, 'model') else (lambda c, k: c[k])
    # feature widths come from the checkpoint's featurisers like the reference (scripts/sample_diffusion.py:140-160):
    # protein = 6 elements + 20 residue types + backbone flag, ligand = class count of data.transform.ligand_atom_mode
    try:
        mode = get(get(get(tc, 'data'), 'transform'), 'ligand_atom_mode')
    except (AttributeError, KeyError, TypeError):
        mode = 'add_aromatic'
    if mode not in LIGAND_ATOM_MODE_CLASSES:
        raise NotImplementedError('checkpoint ligand_atom_mode=%r (known: %s)' % (mode, sorted(LIGAND_ATOM_MODE_CLASSES)))
    model = ScorePosNet3D(get(tc, 'model'), PROTEIN_FEATURE_DIM, LIGAND_ATOM_MODE_CLASSES[mode])
    model.ligand_atom_mode = mode
    if rank == 0:
        model.load_state_dict(ckpt['model'])
    model = model.to(device)
    tdist.broadcast_state_dict(model, src=0)
    return model


def _time_seq(config, model):
    """The time sequence `sample.respaced_steps` asks for (config.sampling_time_seq), or None for the default chain."""
    if config.sample.get('respaced_steps') is None:
        return None
    return sampling_time_seq(config.sample, model.num_timesteps)


def list_pockets(pocket_dir=None, pocket_list=None):
    """Task list in a sharding-independent order: sorted *.pdb of a directory, or the lines of a list file."""
    if (pocket_dir is None) == (pocket_list is None):
        raise ValueError('give exactly one of --pocket_dir / --pocket_list')
    if pocket_dir is not None:
        paths = sorted(os.path.join(pocket_dir, f) for f in os.listdir(pocket_dir) if f.lower().endswith('.pdb'))
    else:
        base = os.path.dirname(os.path.abspath(pocket_list))
        with open(pocket_list) as f:
            paths = [ln.strip() for ln in f if ln.strip() and not ln.startswith('#')]
        paths = [p if os.path.isabs(p) else os.path.join(base, p) for p in paths]
    if not paths:
        raise ValueError('no pockets found')
    return paths


def assign_pockets(paths, rank, world, schedule='round_robin', data_id=None):
    """Pocket ids this rank works on.  round_robin = the reference's `i % NODE_ALL == NODE_THIS`
    (scripts/batch_sample_diffusion.sh:15-21); longest_first balances by ATOM-record count (cost ~ nodes x k)."""
    from . import dist as tdist
    ids = list(range(len(paths)))
    if data_id is not None:
        if not 0 <= data_id < len(paths):
            raise ValueError('data_id %d outside 0..%d' % (data_id, len(paths) - 1))
        return [data_id] if data_id % world == rank else []
    if schedule == 'round_robin':
        return tdist.shard_round_robin(ids, rank, world)
    if schedule == 'longest_first':
        costs = []
        for p in paths:
            with open(p) as f:
                costs.append(sum(1 for ln in f if ln.startswith('ATOM')))
        return tdist.shard_longest_first(costs, world)[rank]
    raise ValueError('schedule %r' % (schedule,))


def sample_pockets(argv):
    from . import dist as tdist
    ap = argparse.ArgumentParser(prog='targetdiff_b200.cli sample_pockets')
    ap.add_argument('config', type=str)
    ap.add_argument('--pocket_dir', type=str)
    ap.add_argument('--pocket_list', type=str)
    ap.add_argument('-i', '--data_id', type=int)
    ap.add_argument('--schedule', type=str, default='round_robin', choices=('round_robin', 'longest_first'))
    ap.add_argument('--device', type=str)
    ap.add_argument('--batch_size', type=int, default=100)
    ap.add_argument('--result_path', type=str, default='./outputs')
    ap.add_argument('--num_samples', type=int)
    a = ap.parse_args(argv)
    config = load_config(a.config)
    sampling_start(config.sample, None, False)      # start ligands are sample_for_pocket's only: refuses sample.start_time
    check_resampling(config.sample, False)          # so is resampling, which needs held atoms: refuses sample.resamplings
    clash_radius, clash_strength = sample_clash_guidance(config.sample)
    connect_radius, connect_length, connect_strength = sample_connect_guidance(config.sample)
    rank, world, local_rank = tdist.init_from_env()
    device = a.device or 'cuda:%d' % local_rank
    paths = list_pockets(a.pocket_dir, a.pocket_list)
    mine = assign_pockets(paths, rank, world, a.schedule, a.data_id)
    model = _load_model(config, device, rank)
    allowed = _allowed_classes(config, model)
    time_seq = _time_seq(config, model)
    num_steps = config.sample.num_steps if time_seq is None else None
    n = a.num_samples if a.num_samples is not None else config.sample.num_samples
    os.makedirs(a.result_path, exist_ok=True)
    if rank == 0:
        shutil.copyfile(a.config, os.path.join(a.result_path, 'sample.yml'))
    done = []
    for i in mine:
        seed_all(config.sample.seed)          # the reference starts one process per pocket, each seeded the same way (:133)
        data = pdb_to_pocket_data(paths[i])
        outputs = sample_diffusion_ligand(model, data, n, batch_size=a.batch_size, device=device, num_steps=num_steps,
                                          pos_only=config.sample.pos_only, center_pos_mode=config.sample.center_pos_mode,
                                          sample_num_atoms=config.sample.sample_num_atoms, time_seq=time_seq,
                                          clash_radius=clash_radius, clash_strength=clash_strength, allowed_types=allowed,
                                          connect_radius=connect_radius, connect_length=connect_length, connect_strength=connect_strength)
        result = add_allowed_classes(add_clash_guidance(build_result(data, outputs), clash_radius, clash_strength), allowed)
        result = add_connect_guidance(result, connect_radius, connect_length, connect_strength)
        result = add_connect_guidance(result, connect_radius, connect_length, connect_strength)
        if time_seq is not None:
            result['time_seq'] = time_seq
        torch.save(result, os.path.join(a.result_path, 'result_%d.pt' % i))
        done.append((i, len(outputs[0]), sum(outputs[-1])))
        print('[rank %d/%d] pocket %d (%s): %d molecules, %.1f s' % (rank, world, i, os.path.basename(paths[i]), done[-1][1], done[-1][2]))
    return done


def _load_ligand_file(path, option):
    """(entries dict, pos float32 [n,3], v int64 [n]) from a .pt (a dict) or .npz file with entries 'pos' and 'v'."""
    if path.endswith('.npz'):
        import numpy as np
        with np.load(path) as z:
            d = {k: z[k] for k in z.files}
    elif path.endswith('.pt'):
        d = torch.load(path, map_location='cpu', weights_only=True)
    else:
        raise ValueError('%s %s: expected a .pt or .npz file' % (option, path))
    if not isinstance(d, dict) or 'pos' not in d or 'v' not in d:
        raise ValueError("%s %s must hold 'pos' [n,3] and 'v' [n]" % (option, path))
    pos = torch.as_tensor(d['pos']).float()
    v = torch.as_tensor(d['v'])
    if v.is_floating_point() or pos.dim() != 2 or pos.shape[1] != 3 or v.dim() != 1 or v.shape[0] != pos.shape[0] or v.shape[0] < 1:
        raise ValueError("%s %s: 'pos' must be [n,3] and 'v' [n] integer class indices (n >= 1), got %s and %s %s"
                         % (option, path, tuple(pos.shape), tuple(v.shape), v.dtype))
    return d, pos, v.long()


def load_fragment(path):
    """(pos float32 [n,3], v int64 [n]) from a .pt (a dict) or .npz file with entries 'pos' and 'v'."""
    _, pos, v = _load_ligand_file(path, '--fragment')
    return pos, v


def load_start_ligand(path):
    """(pos float32 [n,3], v int64 [n], keep int64 [k] or None) from a .pt (a dict) or .npz file with entries 'pos', 'v' and an
    optional 'keep' of atom indices to keep (sample_diffusion_ligand checks their range and uniqueness)."""
    d, pos, v = _load_ligand_file(path, '--start_ligand')
    keep = d.get('keep')
    if keep is not None:
        keep = torch.as_tensor(keep)
        if keep.is_floating_point() or keep.is_complex() or keep.dtype == torch.bool or keep.dim() != 1:
            raise ValueError("--start_ligand %s: 'keep' must be a 1-D array of integer atom indices, got %s %s"
                             % (path, tuple(keep.shape), keep.dtype))
        keep = keep.long()
    return pos, v, keep


def sample_for_pocket(argv):
    ap = argparse.ArgumentParser(prog='targetdiff_b200.cli sample_for_pocket')
    ap.add_argument('config', type=str)
    ap.add_argument('--pdb_path', type=str, required=True)
    ap.add_argument('--device', type=str, default='cuda:0')
    ap.add_argument('--batch_size', type=int, default=100)
    ap.add_argument('--result_path', type=str, default='./outputs_pdb')
    ap.add_argument('--num_samples', type=int)
    ap.add_argument('--fragment', type=str, help=".pt / .npz with 'pos' [n,3] and 'v' [n]: every sample grows from this fragment")
    ap.add_argument('--start_ligand', type=str, help=".pt / .npz with 'pos' [n,3], 'v' [n] and optional 'keep' [k]: every sample starts "
                                                     "from this ligand noised to sample.start_time")
    a = ap.parse_args(argv)
    if a.fragment and a.start_ligand:
        raise ValueError('--fragment cannot be combined with --start_ligand: keep atoms of the start ligand with its \'keep\' entry')
    config = load_config(a.config)
    fragment = load_fragment(a.fragment) if a.fragment else None
    start = load_start_ligand(a.start_ligand) if a.start_ligand else None
    held = fragment is not None or (start is not None and start[2] is not None and len(start[2]) > 0)
    check_resampling(config.sample, held)
    clash_radius, clash_strength = sample_clash_guidance(config.sample)
    connect_radius, connect_length, connect_strength = sample_connect_guidance(config.sample)
    seed_all(config.sample.seed)
    model = _load_model(config, a.device)
    allowed = _allowed_classes(config, model)
    start_time, start_seq = sampling_start(config.sample, model.num_timesteps, start is not None)
    time_seq = _time_seq(config, model) if start is None else start_seq
    T = model.num_timesteps
    base = time_seq if time_seq is not None else list(range(T - 1, T - 1 - int(config.sample.get('num_steps') or T), -1))
    time_path = sampling_time_path(config.sample, T, base, held)
    data = pdb_to_pocket_data(a.pdb_path)
    n = a.num_samples if a.num_samples is not None else config.sample.num_samples
    kw = {} if start is None else dict(start_ligand=start[:2], start_time=start_time, keep_atoms=start[2])
    if time_path is not None:
        kw['time_path'] = time_path
    outputs = sample_diffusion_ligand(model, data, n, batch_size=a.batch_size, device=a.device,
                                      num_steps=config.sample.num_steps if time_seq is None and time_path is None else None,
                                      pos_only=config.sample.pos_only, center_pos_mode=config.sample.center_pos_mode,
                                      sample_num_atoms=config.sample.sample_num_atoms, fixed_ligand=fragment,
                                      time_seq=time_seq if time_path is None else None, clash_radius=clash_radius,
                                      clash_strength=clash_strength, allowed_types=allowed, connect_radius=connect_radius,
                                      connect_length=connect_length, connect_strength=connect_strength, **kw)
    os.makedirs(a.result_path, exist_ok=True)
    shutil.copyfile(a.config, os.path.join(a.result_path, 'sample.yml'))
    result = add_allowed_classes(add_clash_guidance(build_result(data, outputs), clash_radius, clash_strength), allowed)
    result = add_connect_guidance(result, connect_radius, connect_length, connect_strength)
    if fragment is not None:
        result['fixed_ligand_atoms'] = int(fragment[1].shape[0])
    if start is not None:
        result['start_ligand'] = (start[0], start[1])
        result['start_time'] = start_time
        result['kept_atoms'] = [] if start[2] is None else start[2].tolist()
        if config.sample.get('respaced_steps') is not None:
            result['time_seq'] = time_seq
    elif time_seq is not None:
        result['time_seq'] = time_seq
    if time_path is not None:
        result['time_path'] = time_path
    torch.save(result, os.path.join(a.result_path, 'sample.pt'))
    print('Sample done! %d molecules, %.1f s' % (len(outputs[0]), sum(outputs[-1])))


def score_ligands(argv):
    ap = argparse.ArgumentParser(prog='targetdiff_b200.cli score_ligands')
    ap.add_argument('config', type=str)
    ap.add_argument('--pdb_path', type=str, help='the pocket of the --ligand files')
    ap.add_argument('--ligand', type=str, nargs='+', help=".pt / .npz files with 'pos' [n,3] (lab frame) and 'v' [n]")
    ap.add_argument('--samples', type=str, help='a sample.pt / result_{i}.pt: every molecule, in that file\'s own pocket')
    ap.add_argument('--time_steps', type=str, default='10', help="N evenly spaced timesteps (i * T // N), or 'all' for every timestep")
    ap.add_argument('--batch_size', type=int, default=640, help='(ligand, timestep) graphs per engine call')
    ap.add_argument('--embedding', action='store_true', help='also store pred_ligand_v, final_h and final_ligand_h')
    ap.add_argument('--result_path', type=str, default='./outputs_scores')
    ap.add_argument('--device', type=str, default='cuda:0')
    a = ap.parse_args(argv)
    if bool(a.ligand) == bool(a.samples):
        raise ValueError('give either --ligand FILE [FILE ...] (with --pdb_path) or --samples RESULT.pt, not both')
    if a.ligand and not a.pdb_path:
        raise ValueError('--ligand needs --pdb_path')
    if a.samples and a.pdb_path:
        raise ValueError('--samples scores in the pocket stored in the file: --pdb_path is not used with it')
    config = load_config(a.config)
    if a.ligand:
        ligands = [_load_ligand_file(p, '--ligand')[1:] for p in a.ligand]
        sources = [{'source': p} for p in a.ligand]
        data = pdb_to_pocket_data(a.pdb_path)
    else:
        r = torch.load(a.samples, map_location='cpu', weights_only=False)
        data = r['data']
        ligands = list(zip(r['pred_ligand_pos'], r['pred_ligand_v']))
        sources = [{'source': a.samples, 'sample_index': i} for i in range(len(ligands))]
    seed_all(config.sample.seed)
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())          # the likelihood stream's key, drawn before loading the model
    model = _load_model(config, a.device)
    if a.embedding and model.time_emb_dim > 0:
        raise ValueError('--embedding needs a checkpoint without a time embedding (the reference fetch_embedding cannot run either)')
    T = model.num_timesteps
    time_steps = likelihood_time_steps(T, T if a.time_steps == 'all' else int(a.time_steps))
    scores = ligand_nll(model, data, ligands, time_steps=time_steps, batch_size=a.batch_size, device=a.device, seed=seed,
                        embedding=a.embedding)
    out = []
    for src, sc in zip(sources, scores):
        d = {'kl_pos': sc['kl_pos'], 'kl_v': sc['kl_v'], 'nll': sc['nll']}
        for k in ('pred_ligand_v', 'final_h', 'final_ligand_h'):
            if k in sc:
                d[k] = sc[k]
        d.update(src)
        out.append(d)
    os.makedirs(a.result_path, exist_ok=True)
    torch.save(out, os.path.join(a.result_path, 'scores.pt'))
    print('Scored %d ligands at %d timesteps' % (len(out), len(time_steps)))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    commands = {'sample_for_pocket': sample_for_pocket, 'sample_pockets': sample_pockets, 'score_ligands': score_ligands}
    if not argv or argv[0] not in commands:
        raise SystemExit(__doc__)
    commands[argv[0]](argv[1:])


if __name__ == '__main__':
    main()
