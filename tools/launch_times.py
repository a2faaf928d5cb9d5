"""Per-kernel device time of eager denoising steps of a bench workload, from torch.profiler (CUDA activities).

    python tools/launch_times.py --workload cfg3 --steps 3 --out DIR

The engine runs with TDIFF_NO_GRAPH=1, so every launch is its own profiler event.  After `--warmup` unprofiled steps, `--steps`
steps run under the profiler; DIR/launch_times.csv and DIR/launch_times.json list, per kernel name (template arguments included,
so the folded key launch `edge_mlp_v4_kernel<128, true>` is told apart from the value launch `<128, false>`), the launch count,
total and per-step device time and the share of all kernel time.  Kernel times come from the CUDA activity records, not from
host clocks.  Tracing adds host overhead between launches, so step times are for bench.py; this script splits the device time.
"""
import argparse
import collections
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ['TDIFF_NO_GRAPH'] = '1'          # read once when the engine is created


def main():
    import bench
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='cfg3', choices=sorted(bench.WORKLOADS))
    ap.add_argument('--steps', type=int, default=3, help='profiled denoising steps')
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', required=True, help='output directory')
    a = ap.parse_args()
    for k, v in bench.WORKLOADS[a.workload].items():
        setattr(a, k, v)

    import torch
    from torch.profiler import ProfilerActivity, profile
    from targetdiff_b200 import _lib
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    from oracle import synth
    if not torch.cuda.is_available():
        raise SystemExit('launch_times.py needs a CUDA device')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    lib = _lib.load()

    cfg = default_model_config()
    cfg.knn = a.knn
    model = ScorePosNet3D(cfg, synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    model.load_state_dict(synth.make_state_dict(0, {'knn': a.knn}, schedules={k: getattr(model, k).data for k in synth.SCHEDULE_KEYS}),
                          strict=True)
    model = model.to(dev)
    b, G, N, Nl = bench.make_workload(a, 0)
    d = {k: v.to(dev) for k, v in b.items()}
    eng = model.engine(dev)
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    model._bind(eng, d['protein_pos'], d['protein_v'], d['batch_protein'], d['batch_ligand'], 1)
    _lib.check(lib.tdiff_set_ligand(eng, ctypes.c_void_p(d['init_ligand_pos'].data_ptr()), ctypes.c_void_p(d['init_ligand_v'].data_ptr()), 1, st))
    K = synth.LIGAND_NUM_CLASSES
    S = max(a.steps, a.warmup, 1)
    traj = (torch.empty(S, Nl, 3, device=dev), torch.empty(S, Nl, dtype=torch.int64, device=dev),
            torch.empty(S, Nl, K, device=dev), torch.empty(S, Nl, K, device=dev))
    PT = lambda t: ctypes.c_void_p(t.data_ptr())

    def chain(steps, seed):
        _lib.check(lib.tdiff_sample(eng, steps, None, None, ctypes.c_uint64(seed), PT(traj[0]), PT(traj[1]), PT(traj[2]), PT(traj[3]), 0, st))

    chain(max(1, a.warmup), 1)
    torch.cuda.synchronize(dev)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        chain(a.steps, 2)
        torch.cuda.synchronize(dev)

    agg = collections.OrderedDict()
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.time_range.elapsed_us()
        n_t = agg.setdefault(ev.name, [0, 0.0])
        n_t[0] += 1
        n_t[1] += us
    total = sum(t for _, t in agg.values())
    rows = [dict(kernel=k, launches=n, total_us=round(t, 1), us_per_step=round(t / a.steps, 1), avg_us=round(t / n, 2),
                 share=round(t / total, 4) if total else 0.0) for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])]
    gpu = torch.cuda.get_device_name(dev)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'launch_times.csv'), 'w') as f:
        f.write('kernel,launches,total_us,us_per_step,avg_us,share\n')
        for r in rows:
            f.write('"%s",%d,%.1f,%.1f,%.2f,%.4f\n' % (r['kernel'], r['launches'], r['total_us'], r['us_per_step'], r['avg_us'], r['share']))
    summary = dict(workload=bench.workload_name(a), gpu=gpu, profiled_steps=a.steps, kernel_us_per_step=round(total / a.steps, 1), kernels=rows)
    with open(os.path.join(a.out, 'launch_times.json'), 'w') as f:
        json.dump(summary, f, indent=1)
    print('%s, %s: %.1f us of kernel time per step' % (summary['workload'], gpu, total / a.steps))
    for r in rows[:12]:
        print('  %-60s %5d  %10.1f us/step  %6.2f %%' % (r['kernel'][:60], r['launches'], r['us_per_step'], 100 * r['share']))


if __name__ == '__main__':
    main()
