"""Call sequences on one engine handle, through the C-ABI (run with -m gpu; `pytest -s` prints what each sequence compared).

The other GPU tests make one call on a freshly bound batch.  A caller of include/tdiff.h may instead bind once and alternate
tdiff_set_ligand / tdiff_forward, run chains back to back, or rebind the same handle to another batch, and that is where the engine
keeps state between calls: the incremental edge gate (src_prev and the keep marks in etype), the ligand-free feature cache, the
protein-only k-NN keys, the fixed set, the start time and the borrowed tapes, and device buffers that only grow (a batch bound after a
larger one runs on over-sized buffers that still hold the larger batch's data).

Each test runs one sequence of calls on one handle and keeps every output.  Then every call that produced an output is replayed on a
fresh engine: create, bind the same batch, set the ligand state the call saw (tdiff_get_ligand just before it), set the same fixed
set / start / time, and make that one call.  Every cache is exact, so the reused engine runs the same kernels on the same values, and
the two must agree bit for bit: pred_pos, logits, final_h, edge_index and e_w of a forward; the four trajectories, the final state,
edge_index and e_w of a chain.  One anchor per sequence against the CPU oracle (restate.forward, or the oracle chain on the same
tapes, at the tolerances of test_gpu_configs.py) catches both runs being equally wrong.  Only one engine is alive at a time."""
import ctypes

import pytest
import torch

from oracle import fixed_atoms, restate, start_ligand, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
K13 = synth.LIGAND_NUM_CLASSES
POS_RTOL, POS_ATOL, LOGIT_ATOL, H_TOL = 1e-4, 1e-5, 1e-3, 1e-4
HYBRID = {'cutoff_mode': 'hybrid', 'knn': 24}
CONFIGS = {'default': None, 'ew_r': {'ew_net_type': 'r'}, 'blocks2': {'num_blocks': 2},
           'time_emb': {'time_emb_dim': 1, 'time_emb_mode': 'simple'}, 'hybrid': HYBRID}


def _vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _lib():
    from targetdiff_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------ batches
class Batch:
    """A ragged batch on the device.  `wall`: each graph's ligand moved from the pocket centre towards the pocket wall by this fraction
    of the pocket's radius, so that protein atoms on the far side have no ligand atom within two hops of the k-NN graph: those are the
    rows the ligand-free cache restores (with the ligand at the centre every protein atom of these small pockets is touched)."""

    def __init__(self, seed, pcs, lcs, wall=0.0):
        self.pc, self.lc = list(pcs), list(lcs)
        self.cpu = c = synth.make_ragged_batch(seed, pcs, lcs)
        for g in range(len(pcs)):
            p, sel = c['protein_pos'][c['batch_protein'] == g], c['batch_ligand'] == g
            if len(p):
                c['init_ligand_pos'][sel] += torch.tensor([wall, 0.0, 0.0]) * float((p - p.mean(0)).norm(dim=1).max())
        self.ppos = c['protein_pos'].to(DEV).contiguous()
        self.pfeat = c['protein_v'].float().to(DEV).contiguous()
        self.lpos = c['init_ligand_pos'].to(DEV).contiguous()
        self.lv = c['init_ligand_v'].to(DEV).contiguous()
        self.B, self.Np, self.Nl = len(self.pc), sum(self.pc), sum(self.lc)
        self.N = self.Np + self.Nl

    def ligand_node(self):
        """[N] bool: which composed-order nodes are ligand atoms."""
        m = []
        for p, l in zip(self.pc, self.lc):
            m += [False] * p + [True] * l
        return torch.tensor(m)

    def pocket_centres(self):
        return torch.stack([self.cpu['protein_pos'][self.cpu['batch_protein'] == g].mean(0) for g in range(self.B)]).to(DEV)


def _batches(cfg_name):
    """A, B and C have more than k = 32 protein atoms in every graph (the ligand-free cache is on); the small batch has one graph of
    at most k nodes (the cache is off, and rows have absent neighbour slots)."""
    A = Batch(11, [90, 120, 80, 110], [9, 14, 5, 11], wall=0.8)
    Bsame = Batch(12, [90, 120, 80, 110], [9, 14, 5, 11], wall=0.8)    # A's counts, other coordinates and features
    C = Batch(13, [130, 150, 120, 140], [20, 25, 12, 30], wall=0.8)    # larger: buffers grow (and are poison-filled)
    if cfg_name == 'hybrid':        # hybrid needs >= k protein atoms beside a ligand; the <= k graph has none
        small = Batch(14, [40, 24, 45], [9, 0, 11])
    else:
        small = Batch(14, [40, 20, 45], [9, 6, 11])
    return A, Bsame, C, small


def _moved(b):
    """The batch's ligand moved so that protein neighbour lists change: graph 0 reflected through its pocket centre, graph 1 shifted
    4 A onto another patch of the pocket wall, graph 2 jittered by 0.05 A (same neighbours, new lengths), the rest as they were."""
    pos = b.lpos.clone()
    ctr = b.pocket_centres()
    bl = b.cpu['batch_ligand'].to(DEV)
    g = torch.Generator().manual_seed(3)
    jit = (torch.randn(b.Nl, 3, generator=g) * 0.05).to(DEV)
    for a in range(b.Nl):
        gi = int(bl[a])
        if gi == 0:
            pos[a] = 2 * ctr[0] - pos[a]
        elif gi == 1:
            pos[a] = pos[a] + torch.tensor([-4.0, -1.0, 0.5], device=DEV)
        elif gi == 2:
            pos[a] = pos[a] + jit[a]
    return pos.contiguous()


def _tape(seed, S, n, K=K13):
    pn, vu = synth.make_tape(seed, S, n, K)
    return pn.to(DEV).contiguous(), vu.to(DEV).contiguous()


# ------------------------------------------------------------------------------------------------ one handle, its log, the replay
class Seq:
    """Drives one engine handle through the C-ABI and logs every output-producing call with what a fresh engine needs to replay it."""

    def __init__(self, cfg_name, weight_seed=0):
        from targetdiff_b200.config import default_model_config
        from targetdiff_b200.score_model import ScorePosNet3D
        cfg = CONFIGS.get(cfg_name, cfg_name) if isinstance(cfg_name, str) else cfg_name
        self.cfg = cfg
        c = default_model_config()
        c.update(cfg or {})
        self.sd = synth.make_state_dict(weight_seed, cfg, schedules=restate.make_schedules(cfg))
        m = ScorePosNet3D(c, synth.PROTEIN_FEATURE_DIM, K13)
        m.load_state_dict(self.sd, strict=True)
        self.model = m.to(DEV)
        self.time_emb = c.time_emb_dim > 0
        self.T = int(self.sd['betas'].shape[0])
        self.lib = _lib().load()
        self.log = []
        self.fresh()

    # -- plumbing
    def fresh(self):
        self.model._drop_engine()
        self.eng = self.model.engine(DEV)
        self.batch, self.mode, self.fixed, self.fixed_tape, self.start = None, None, None, (None, None), None

    def close(self):
        self.model._drop_engine()

    def st(self):
        return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)

    def ok(self, rc):
        _lib().check(rc)

    # -- state-setting calls
    def bind(self, b, mode=1):
        L = _lib()
        rc = self.lib.tdiff_bind_batch(self.eng, b.B, L.i32_array(b.pc), L.i32_array(b.lc), _vp(b.ppos), _vp(b.pfeat), mode, self.st())
        if rc == 0:
            self.batch, self.mode, self.fixed, self.fixed_tape, self.start = b, mode, None, (None, None), None
        return rc

    def set_ligand(self, pos, v, apply_center=1):
        return self.lib.tdiff_set_ligand(self.eng, _vp(pos), _vp(v), apply_center, self.st())

    def set_fixed(self, mask, pos0=None, v0=None, apply_center=1):
        rc = self.lib.tdiff_set_fixed(self.eng, _vp(mask), _vp(pos0), _vp(v0), apply_center, self.st())
        if rc == 0:
            self.fixed = None if mask is None else (mask, pos0, v0, apply_center)
        return rc

    def set_fixed_tape(self, pn, vu):
        self.ok(self.lib.tdiff_set_fixed_tape(self.eng, _vp(pn), _vp(vu)))
        self.fixed_tape = (pn, vu)

    def set_start(self, t0, pn=None, vu=None):
        rc = self.lib.tdiff_set_start(self.eng, t0, _vp(pn), _vp(vu))
        if rc == 0:
            self.start = None if t0 < 0 else (t0, pn, vu)
        return rc

    def get_ligand(self, add_offset=0):
        n = self.batch.Nl
        pos, v = torch.empty(n, 3, device=DEV), torch.empty(n, dtype=torch.int64, device=DEV)
        self.ok(self.lib.tdiff_get_ligand(self.eng, _vp(pos), _vp(v), add_offset, self.st()))
        return pos, v

    def offset(self):
        off = torch.empty(self.batch.B, 3, device=DEV)
        self.ok(self.lib.tdiff_get_offset(self.eng, _vp(off), self.st()))
        return off

    def _graph(self):
        E = self.lib.tdiff_num_edges(self.eng, self.st())
        assert E >= 0, _lib().last_error()
        ei, ew = torch.empty(2, E, dtype=torch.int64, device=DEV), torch.empty(E, device=DEV)
        self.ok(self.lib.tdiff_get_edge_index(self.eng, _vp(ei), self.st()))
        self.ok(self.lib.tdiff_get_edge_weight(self.eng, _vp(ew), self.st()))
        return ei, ew

    # -- output-producing calls (logged)
    def _forward(self, fix_x, t):
        b = self.batch
        if self.time_emb:
            tn = torch.full((b.B,), float(t), device=DEV)
            tn = (tn / torch.full_like(tn, float(self.T))).contiguous()
            self.ok(self.lib.tdiff_set_time(self.eng, _vp(tn), self.st()))
        out = {'pred_pos': torch.empty(b.Nl, 3, device=DEV), 'logits': torch.empty(b.Nl, K13, device=DEV),
               'final_h': torch.empty(b.N, 128, device=DEV)}
        self.ok(self.lib.tdiff_forward(self.eng, _vp(out['pred_pos']), _vp(out['logits']), _vp(out['final_h']), fix_x, self.st()))
        out['edge_index'], out['e_w'] = self._graph()
        return out

    def _chain(self, S, seq, tape, seed, pos_only):
        n = self.batch.Nl
        out = {'pos_traj': torch.empty(S, n, 3, device=DEV), 'v_traj': torch.empty(S, n, dtype=torch.int64, device=DEV),
               'v0_traj': torch.empty(S, n, K13, device=DEV), 'vt_traj': torch.empty(S, n, K13, device=DEV)}
        pn, vu = tape if tape is not None else (None, None)
        a = (_vp(pn), _vp(vu), ctypes.c_uint64(seed), _vp(out['pos_traj']), _vp(out['v_traj']), _vp(out['v0_traj']), _vp(out['vt_traj']),
             int(pos_only), self.st())
        if seq is None:
            self.ok(self.lib.tdiff_sample(self.eng, S, *a))
        else:
            self.ok(self.lib.tdiff_sample_seq(self.eng, _lib().i32_array(seq), S, *a))
        out['pos'], out['v'] = self.get_ligand(1)
        out['edge_index'], out['e_w'] = self._graph()
        return out

    def _record(self, label, kind, args, out):
        pre = self._pre
        self.log.append(dict(label=label, kind=kind, args=args, out=out, batch=self.batch, mode=self.mode, fixed=self.fixed,
                             fixed_tape=self.fixed_tape, start=self.start, pre=pre))
        return out

    def forward(self, label, fix_x=0, t=500):
        self._pre = self.get_ligand(0)
        return self._record(label, 'forward', (fix_x, t), self._forward(fix_x, t))

    def chain(self, label, S=None, seq=None, tape=None, seed=1, pos_only=0):
        S = len(seq) if seq is not None else S
        self._pre = self.get_ligand(0)
        return self._record(label, 'chain', (S, seq, tape, seed, pos_only), self._chain(S, seq, tape, seed, pos_only))

    # -- replay
    def replay(self, ent, pre=None):
        """The logged call on a fresh engine: bind, the ligand state it saw (or `pre`), fixed set / tape / start, the call."""
        self.fresh()
        self.ok(self.bind(ent['batch'], ent['mode']))
        pos, v = ent['pre'] if pre is None else pre
        self.ok(self.set_ligand(pos, v, 0))
        if ent['fixed'] is not None:
            self.ok(self.set_fixed(*ent['fixed']))
            self.set_fixed_tape(*ent['fixed_tape'])
        if ent['start'] is not None:
            self.ok(self.set_start(*ent['start']))
        if ent['kind'] == 'forward':
            return self._forward(*ent['args'])
        return self._chain(*ent['args'])

    def check_replays(self, name):
        """Every logged output against its fresh-engine replay, bit for bit."""
        bad = []
        log, self.log = self.log, []
        for ent in log:
            ref = self.replay(ent)
            for k, got in ent['out'].items():
                want = ref[k]
                if got.shape != want.shape or not torch.equal(got, want):
                    d = float((got.double() - want.double()).abs().max()) if got.shape == want.shape else float('nan')
                    bad.append('%s: %s differs (shape %s vs %s, max |diff| %.3g)' % (ent['label'], k, tuple(got.shape), tuple(want.shape), d))
        print('%s: %d calls replayed on fresh engines, %d outputs differ' % (name, len(log), len(bad)))
        assert not bad, '\n'.join(bad)
        return log

    # -- oracle anchors
    def anchor_forward(self, ent):
        b = ent['batch']
        c = b.cpu
        self.fresh()
        self.ok(self.bind(b, ent['mode']))
        off = self.offset().cpu()
        pp = c['protein_pos'] - off[c['batch_protein']]
        lp, lv = ent['pre'][0].cpu(), ent['pre'][1].cpu()
        fix_x, t = ent['args']
        kw = {'time_step': torch.full((b.B,), t, dtype=torch.long)} if self.time_emb else {}
        tr = {}
        want = restate.forward(self.sd, self.cfg, pp, c['protein_v'], c['batch_protein'], lp, lv, c['batch_ligand'], fix_x=bool(fix_x),
                               trace=tr, **kw)
        got = ent['out']
        torch.testing.assert_close(got['pred_pos'].cpu(), want['pred_ligand_pos'], rtol=POS_RTOL, atol=POS_ATOL)
        torch.testing.assert_close(got['logits'].cpu(), want['pred_ligand_v'], rtol=0, atol=LOGIT_ATOL)
        torch.testing.assert_close(got['final_h'].cpu(), want['final_h'], rtol=H_TOL, atol=H_TOL)
        if (self.cfg or {}).get('num_blocks', 1) == 1 and (self.cfg or {}).get('cutoff_mode', 'knn') == 'knn':
            assert torch.equal(got['edge_index'].cpu(), tr['edge_index'])
        print('%s: oracle forward, max |pred_pos - oracle| %.2e' % (ent['label'], float((got['pred_pos'].cpu() - want['pred_ligand_pos']).abs().max())))


def _check_chain_vs_oracle(label, got, want):
    v = torch.stack(want['v_traj'])
    first_bad = (got['v_traj'].cpu() != v).any(1).nonzero()
    assert len(first_bad) == 0, '%s: atom types diverge from the oracle at step %d' % (label, int(first_bad[0]))
    torch.testing.assert_close(got['pos_traj'].cpu(), torch.stack(want['pos_traj']), rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['pos'].cpu(), want['pos'], rtol=POS_RTOL, atol=POS_ATOL)
    torch.testing.assert_close(got['v0_traj'].cpu(), torch.stack(want['v0_traj']), rtol=0, atol=LOGIT_ATOL)
    torch.testing.assert_close(got['vt_traj'].cpu(), torch.stack(want['vt_traj']), rtol=0, atol=LOGIT_ATOL)
    print('%s: oracle chain, max |pos - oracle| %.2e' % (label, float((got['pos_traj'].cpu() - torch.stack(want['pos_traj'])).abs().max())))


def _cpu_args(b):
    c = b.cpu
    return c['protein_pos'], c['protein_v'], c['batch_protein'], c['init_ligand_pos'], c['init_ligand_v'], c['batch_ligand']


# ------------------------------------------------------------------------------------------------ 1. set_ligand / forward
def _seq_forwards(s, A):
    s.ok(s.bind(A, 1))
    s.ok(s.set_ligand(A.lpos, A.lv, 1))
    f0 = s.forward('forward, first')
    s.ok(s.set_ligand(_moved(A), A.lv, 1))
    f1 = s.forward('forward, ligand moved')
    g = torch.Generator().manual_seed(4)
    s.ok(s.set_ligand((A.lpos + (torch.randn(A.Nl, 3, generator=g) * 0.3).to(DEV)).contiguous(), None, 1))   # types kept
    s.forward('forward, set_ligand(d_v=NULL)')
    s.forward('forward, fix_x=1', fix_x=1)
    s.forward('forward, fix_x=0 on the same state', fix_x=0)
    return f0, f1


def _protein_dst_ligand_edges(b, ei):
    lig = b.ligand_node().to(ei.device)
    sel = lig[ei[0]] & ~lig[ei[1]]
    return set(map(tuple, ei[:, sel].t().tolist()))


@pytest.mark.parametrize('cfg_name', list(CONFIGS))
def test_set_ligand_forward_sequence(cfg_name):
    s = Seq(cfg_name)
    A = _batches(cfg_name)[0]
    f0, f1 = _seq_forwards(s, A)
    # the move changed which ligand atoms sit in protein atoms' neighbour lists (so the edge gate's reuse has work to do)
    assert _protein_dst_ligand_edges(A, f0['edge_index']) != _protein_dst_ligand_edges(A, f1['edge_index'])
    log = s.check_replays('set_ligand/forward [%s]' % cfg_name)
    s.anchor_forward(log[1])
    s.close()


# ------------------------------------------------------------------------------------------------ 2. chains, forward on the cache path
def _seq_chains(s, A, S, noise, tag=''):
    s.ok(s.bind(A, 1))
    s.ok(s.set_ligand(A.lpos, A.lv, 1))
    tape = _tape(21, S, A.Nl) if noise == 'tape' else None
    c1 = s.chain(tag + 'chain 1 (S=%d, %s)' % (S, noise), S=S, tape=tape, seed=2 ** 40 + 7)
    s.forward(tag + 'forward after chain 1 (ligand-free cache built)')
    tape2 = _tape(22, S, A.Nl) if noise == 'tape' else None
    s.chain(tag + 'chain 2 without set_ligand', S=S, tape=tape2, seed=2 ** 40 + 8)
    s.forward(tag + 'forward after chain 2')
    return c1, tape


CHAIN_CASES = [('default', 1, 'tape'), ('default', 2, 'philox'), ('default', 4, 'tape'), ('ew_r', 3, 'tape'), ('blocks2', 3, 'tape'), ('time_emb', 3, 'tape'), ('hybrid', 3, 'tape')]


@pytest.mark.parametrize('cfg_name,S,noise', CHAIN_CASES)
def test_chain_forward_chain_sequence(cfg_name, S, noise):
    """num_steps 1 and 2 run eagerly, >= 3 replay the captured step graph.  The second chain starts from the first one's output (the
    fresh engine gets it through tdiff_get_ligand / tdiff_set_ligand)."""
    s = Seq(cfg_name)
    A = _batches(cfg_name)[0]
    c1, tape = _seq_chains(s, A, S, noise)
    log = s.check_replays('chain/forward/chain [%s, S=%d, %s]' % (cfg_name, S, noise))
    s.anchor_forward(log[1])
    if tape is not None and cfg_name == 'default':
        want = restate.sample_diffusion(s.sd, s.cfg, *_cpu_args(A), tape[0].cpu(), tape[1].cpu(), num_steps=S)
        _check_chain_vs_oracle('chain 1', c1, want)
    s.close()


# ------------------------------------------------------------------------------------------------ 3. fixed set and start
def _mask(b, lead=3):
    m = torch.zeros(b.Nl, dtype=torch.uint8)
    a = 0
    for n in b.lc:
        m[a:a + min(lead, n - 1)] = 1
        a += n
    return m.to(DEV)


@pytest.mark.parametrize('arm,noise', [('fixed', 'tape'), ('fixed', 'philox'), ('start', 'tape'), ('start', 'philox'),
                                       ('start_fixed', 'tape')])
def test_fixed_and_start_persist_across_chains(arm, noise):
    """The fixed set, its tape and an armed start persist until the next bind.  A start-armed chain noises the ligand state it is
    given: the second one, without tdiff_set_ligand, starts from the first chain's output, not from the start ligand."""
    s = Seq('default')
    A = _batches('default')[0]
    t0, seq = 300, [300, 200, 20, 0]
    S = len(seq) if arm.startswith('start') else 3
    tape = lambda sd: _tape(sd, S, A.Nl) if noise == 'tape' else None     # noqa: E731
    s.ok(s.bind(A, 1))
    s.ok(s.set_ligand(A.lpos, A.lv, 1))
    mask = _mask(A)
    ft = st = None
    if arm.endswith('fixed'):
        s.ok(s.set_fixed(mask, A.lpos, A.lv, 1))
        if noise == 'tape':
            ft = _tape(31, S + 1, A.Nl)
            s.set_fixed_tape(*ft)
    if arm.startswith('start'):
        g = torch.Generator().manual_seed(32)
        st = (torch.randn(A.Nl, 3, generator=g).to(DEV), torch.rand(A.Nl, K13, generator=g).to(DEV)) if noise == 'tape' else (None, None)
        s.ok(s.set_start(t0, *st))
    run = (lambda lbl, tp, sd: s.chain(lbl, seq=seq, tape=tp, seed=sd)) if arm.startswith('start') else \
        (lambda lbl, tp, sd: s.chain(lbl, S=S, tape=tp, seed=sd))
    t1 = tape(41)
    c1 = run('chain 1', t1, 51)
    s.forward('forward after chain 1')
    c2 = run('chain 2 without set_ligand', tape(42), 52)
    log = s.check_replays('%s/%s' % (arm, noise))
    if arm.startswith('start'):
        # the contract: chain 2 re-noised chain 1's output.  From the start ligand itself the same chain gives something else.
        other = s.replay(log[2], pre=(log[0]['pre']))
        assert not torch.equal(other['pos_traj'], c2['pos_traj'])
    s.anchor_forward(log[1])
    if noise == 'tape':
        fx = dict(fixed_mask=mask.cpu().bool(), fixed_tape=(ft[0].cpu(), ft[1].cpu())) if ft is not None else {}
        if arm.startswith('start'):
            want = start_ligand.sample_diffusion(s.sd, None, *_cpu_args(A), t1[0].cpu(), t1[1].cpu(), t0, (st[0].cpu(), st[1].cpu()), seq, **fx)
        else:
            want = fixed_atoms.sample_diffusion(s.sd, None, *_cpu_args(A), t1[0].cpu(), t1[1].cpu(), fx['fixed_mask'], fx['fixed_tape'],
                                                num_steps=S)
        _check_chain_vs_oracle('chain 1 (%s)' % arm, c1, want)
    s.close()


# ------------------------------------------------------------------------------------------------ 4. rebinding one handle
@pytest.mark.parametrize('cfg_name', list(CONFIGS))
def test_rebind_sequence(cfg_name):
    """A, then B with A's counts but other protein coordinates and features (nothing is reallocated, every cache must be rebuilt),
    then the larger C (buffers grow), then A again (over-sized buffers holding C's data); then a batch with a graph of at most k
    nodes (the ligand-free cache off) and back; then A with center_mode 0.  Each bind is followed by a chain and a forward."""
    s = Seq(cfg_name)
    A, Bsame, C, small = _batches(cfg_name)
    steps = [(A, 1), (Bsame, 1), (C, 1), (A, 1), (small, 1), (A, 1), (small, 1), (A, 0)]
    offsets = []
    for i, (b, mode) in enumerate(steps):
        s.ok(s.bind(b, mode))
        offsets.append(s.offset())
        s.ok(s.set_ligand(b.lpos, b.lv, 1))
        s.chain('bind %d: chain' % i, S=3, tape=_tape(60 + i, 3, b.Nl))
        s.forward('bind %d: forward' % i)
    log = s.check_replays('rebind [%s]' % cfg_name)
    # the offset: the per-graph protein centroid under center_mode 1, zeros under 0
    for (b, mode), off in zip(steps, offsets):
        if mode == 0:
            assert torch.equal(off, torch.zeros_like(off))
        else:
            c = b.cpu
            want = restate.center_pos(c['protein_pos'], c['init_ligand_pos'], c['batch_protein'], c['batch_ligand'])[2]
            torch.testing.assert_close(off.cpu(), want, rtol=1e-6, atol=1e-6)
    s.anchor_forward(log[7])          # A on the buffers C left behind
    s.anchor_forward(log[15])         # A under center_mode 0
    s.close()


# ------------------------------------------------------------------------------------------------ 6. refusals leave the state usable
def _probe(s, A, mask=None):
    """The calls that are valid on batch A: set the ligand, forward, a 3-step chain (with the fixed set `mask` if given)."""
    s.ok(s.set_ligand(A.lpos, A.lv, 1))
    f = s._forward(0, 500)
    ft = _tape(72, 4, A.Nl)                      # borrowed by the engine: alive until the chain has run
    if mask is not None:
        s.ok(s.set_fixed(mask, A.lpos, A.lv, 1))
        s.set_fixed_tape(*ft)
    c = s._chain(3, None, _tape(71, 3, A.Nl), 1, 0)
    if mask is not None:
        s.ok(s.set_fixed(None))
        s.set_fixed_tape(None, None)
    return f, c


def _same(a, b, what):
    for x, y in zip(a, b):
        for k in x:
            assert torch.equal(x[k], y[k]), '%s: %s differs after the refusal' % (what, k)


@pytest.mark.parametrize('cfg_name', ['default', 'hybrid'])
def test_refusals_leave_the_bound_batch_usable(cfg_name):
    """After each refused call the calls that were valid before give bit-identical outputs.  The refused binds are the ones whose
    checks come after the slot width is known: a graph of more than 2800 nodes, NULL protein arrays beside a larger ligand, and (hybrid)
    k + n_ligand - 1 above 64 slots; a hybrid refusal there must not leave the bound batch with the refused batch's slot width."""
    s = Seq(cfg_name)
    L = _lib()
    A = _batches(cfg_name)[0]
    s.ok(s.bind(A, 1))
    base = _probe(s, A)
    mask = _mask(A)
    fixed_base = _probe(s, A, mask)
    # refused binds (protein arrays of the bound size, so that nothing could be read out of bounds had a bind gone through)
    def bind_counts(pc, lc, null=False):
        ppos, pfeat = torch.zeros(sum(pc), 3, device=DEV), torch.zeros(sum(pc), synth.PROTEIN_FEATURE_DIM, device=DEV)
        return s.lib.tdiff_bind_batch(s.eng, len(pc), L.i32_array(pc), L.i32_array(lc), None if null else _vp(ppos),
                                      None if null else _vp(pfeat), 1, s.st())

    assert bind_counts([2790 if cfg_name == 'hybrid' else 2781], [20]) == L.TDIFF_EINVAL and b'2800' in s.lib.tdiff_last_error()
    _same(_probe(s, A), base, 'bind of a 2801+ node graph')
    assert bind_counts([40, 52, 36, 45], [9, 14, 5, 40], null=True) == L.TDIFF_EINVAL
    assert b'null protein arrays' in s.lib.tdiff_last_error()
    _same(_probe(s, A), base, 'bind with NULL protein arrays')
    if cfg_name == 'hybrid':
        assert bind_counts([40, 52, 36, 45], [9, 14, 5, 50]) == L.TDIFF_EINVAL and b'neighbour slots' in s.lib.tdiff_last_error()
        _same(_probe(s, A), base, 'bind with k + n_ligand - 1 > 64')
    # set_ligand with a class >= K drops the ligand state; setting it again restores everything
    bad_v = A.lv.clone()
    bad_v[3] = K13
    assert s.set_ligand(A.lpos, bad_v, 1) == L.TDIFF_EINVAL
    assert s.lib.tdiff_forward(s.eng, None, None, None, 0, s.st()) == L.TDIFF_ESTATE
    _same(_probe(s, A), base, 'set_ligand with a class >= K')
    # set_fixed with a bad class: refused, and the engine is left without a fixed set
    s.ok(s.set_ligand(A.lpos, A.lv, 1))
    s.ok(s.set_fixed(mask, A.lpos, A.lv, 1))
    bad_v0 = A.lv.clone()
    bad_v0[0] = K13 + 2                 # a masked row
    assert s.set_fixed(mask, A.lpos, bad_v0, 1) == L.TDIFF_EINVAL
    s.ok(s.set_ligand(A.lpos, A.lv, 1))
    c = s._chain(3, None, _tape(71, 3, A.Nl), 1, 0)
    assert all(torch.equal(c[k], base[1][k]) for k in c), 'a refused set_fixed leaves no fixed set'
    _same(_probe(s, A, mask), fixed_base, 'set_fixed with a bad class, then a valid one')
    # sample_seq with a bad sequence, set_start out of range, tdiff_sample with a start armed: the ligand state is untouched
    s.ok(s.set_ligand(A.lpos, A.lv, 1))
    before = s.get_ligand(0)
    T = s.T
    for seq in ([T - 1, T - 1, 0], [T - 2, 10], [T - 1, 5, -1], [T - 1, 20, 40]):
        rc = s.lib.tdiff_sample_seq(s.eng, L.i32_array(seq), len(seq), None, None, ctypes.c_uint64(1), None, None, None, None, 0, s.st())
        assert rc == L.TDIFF_EINVAL
    assert s.set_start(T, None, None) == L.TDIFF_EINVAL
    s.ok(s.set_start(100))
    assert s.lib.tdiff_sample(s.eng, 3, None, None, ctypes.c_uint64(1), None, None, None, None, 0, s.st()) == L.TDIFF_EINVAL
    s.ok(s.set_start(-1))
    after = s.get_ligand(0)
    assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1])
    _same(_probe(s, A), base, 'refused chains')
    s.close()


# ------------------------------------------------------------------------------------------------ 7. a side stream
def test_sequences_on_a_side_stream():
    """Sequences 1 and 2 on a torch side stream (cudaStreamNonBlocking: not ordered after the legacy default stream) against the
    same sequences on the default stream, bit for bit.  Every engine is fresh, so its buffers are allocated (and, in the test suite,
    poison-filled) during the run.  A pass does not prove there is no race: it shows none happened in this run."""
    runs = []
    for side in (False, True):
        s = Seq('default')
        A = _batches('default')[0]
        side_stream = torch.cuda.Stream(DEV)
        side_stream.wait_stream(torch.cuda.current_stream(DEV))
        with torch.cuda.stream(side_stream) if side else torch.cuda.stream(torch.cuda.current_stream(DEV)):
            s.fresh()
            _seq_forwards(s, A)
            s.fresh()
            _seq_chains(s, A, 4, 'tape')
        torch.cuda.synchronize()
        runs.append([e['out'] for e in s.log])
        s.close()
    assert len(runs[0]) == len(runs[1])
    for i, (x, y) in enumerate(zip(*runs)):
        for k in x:
            assert torch.equal(x[k], y[k]), 'call %d: %s differs between the default stream and a side stream' % (i, k)
