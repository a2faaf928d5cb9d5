"""The layer forms of AttentionLayerO2TwoUpdateNodeGeneral (num_x2h, num_h2x, sync_twoup; reference models/uni_transformer.py:143-210)
and forward(..., return_all=True) (models/molopt_score_model.py:360-367) on the CPU side: the restatement against the unmodified
reference (pins of oracle/make_layer_form_pins.py) and, for the default form, against oracle.restate; the one-layer reference against the
restatement; the model's state_dict layout and the configuration checks of the Python surface and of the C-ABI."""
import ctypes
import sys

import pytest
import torch

from oracle import layer_forms, layerwise, refload, restate, synth
from oracle import make_reference_pins as pins_mod
from oracle.make_layer_form_pins import LAYER_FORM_CONFIGS, OUT, RETURN_ALL_BLOCKS, chain_inputs, return_all_inputs
from oracle.make_reference_pins import equal, option_id

if refload.SHIMS not in sys.path:
    sys.path.insert(0, refload.SHIMS)


@pytest.fixture(scope='module')
def pins():
    n = torch.get_num_threads()
    torch.set_num_threads(pins_mod.THREADS)       # the thread count the pins were computed with
    yield torch.load(OUT, weights_only=True)
    torch.set_num_threads(n)


@pytest.mark.parametrize('cfgd', [{}, {'num_blocks': 2, 'ew_net_type': 'r', 'x2h_out_fc': True}, {'cutoff_mode': 'hybrid', 'knn': 8}],
                         ids=lambda c: option_id(c) or 'default')
def test_default_form_equals_restate(cfgd):
    """For the default form (num_x2h = num_h2x = 1, sync_twoup = False) oracle.layer_forms performs oracle.restate's operations: the
    forward (with its trace) and a 3-step chain are bit-identical."""
    sd = synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd))
    b, pn, vu = chain_inputs()
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    want = restate.sample_diffusion(sd, cfgd, *args, pn, vu, num_steps=3)
    got = layer_forms.sample_diffusion(sd, cfgd, *args, pn, vu, num_steps=3)
    for k in ('pos', 'v'):
        assert torch.equal(got[k], want[k]), k
    for k in ('pos_traj', 'v_traj', 'v0_traj', 'vt_traj'):
        assert torch.equal(torch.stack(got[k]), torch.stack(want[k])), k
    b, pp, lp = return_all_inputs()
    fa = (pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'])
    t1, t2 = {}, {}
    want = restate.forward(sd, cfgd, *fa, trace=t1)
    got = layer_forms.forward(sd, cfgd, *fa, trace=t2, return_all=True)
    for k in ('pred_ligand_pos', 'pred_ligand_v', 'final_h', 'final_ligand_h'):
        assert torch.equal(got[k], want[k]), k
    assert all(torch.equal(a, c) for a, c in zip(t1['all_h'] + t1['all_x'], t2['all_h'] + t2['all_x']))
    ref = layer_forms.LayerFormRef.from_trace(sd, cfgd, t1, dtype=torch.float32)
    old = layerwise.LayerRef.from_trace(sd, cfgd, t1, dtype=torch.float32)
    h, x = t1['all_h'][0], t1['all_x'][0]
    assert all(torch.equal(a, c) for a, c in zip(ref(0, h, x), old(0, h, x)))


@pytest.mark.parametrize('cfgd', LAYER_FORM_CONFIGS, ids=option_id)
def test_layer_form_chain_restatement_bit_exact(pins, cfgd):
    """state_dict key order and a 3-step sampling chain of the restatement against the unmodified reference, bit for bit."""
    want = pins[option_id(cfgd)]
    sd = synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd))
    assert equal(list(sd.keys()), want['keys'])
    b, pn, vu = chain_inputs()
    args = (b['protein_pos'], b['protein_v'], b['batch_protein'], b['init_ligand_pos'], b['init_ligand_v'], b['batch_ligand'])
    got = layer_forms.sample_diffusion(sd, cfgd, *args, pn, vu, num_steps=3)
    assert equal(got['pos'], want['pos']) and equal(got['v'], want['v'])
    for k in ('v0_traj', 'vt_traj', 'pos_traj'):
        assert equal(list(got[k]), want[k]), k


@pytest.mark.parametrize('nb', RETURN_ALL_BLOCKS)
@pytest.mark.parametrize('cfgd', LAYER_FORM_CONFIGS, ids=option_id)
def test_layer_form_return_all_restatement_bit_exact(pins, cfgd, nb):
    """forward(..., return_all=True) with num_blocks = nb: the per-block lists (num_blocks + 1 entries) and the final outputs."""
    want = pins[option_id(cfgd)]['return_all_%d' % nb]
    cb = dict(cfgd, num_blocks=nb)
    sd = synth.make_state_dict(1, cb, schedules=restate.make_schedules(cb))
    b, pp, lp = return_all_inputs()
    got = layer_forms.forward(sd, cb, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], return_all=True)
    assert len(got['layer_pred_ligand_pos']) == len(got['layer_pred_ligand_v']) == nb + 1
    for k in ('pred_ligand_pos', 'pred_ligand_v', 'final_h', 'layer_pred_ligand_pos', 'layer_pred_ligand_v'):
        assert equal(got[k], want[k]), k
    assert equal(got['layer_pred_ligand_pos'][-1], want['pred_ligand_pos'])


@pytest.mark.parametrize('cfgd', LAYER_FORM_CONFIGS, ids=option_id)
def test_layer_ref_fp32_chain_is_forward(cfgd):
    """oracle.layer_forms.LayerFormRef at fp32 is layer_forms.forward's own layer for every form, bit for bit (block 0)."""
    sd = synth.make_state_dict(3, cfgd, schedules=restate.make_schedules(cfgd))
    b = synth.make_batch(8, 3, n_protein=60, ligand_sizes=[9, 1, 14])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    layer_forms.forward(sd, dict(cfgd, num_blocks=1), pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    ref = layer_forms.LayerFormRef.from_trace(sd, cfgd, tr, dtype=torch.float32)
    h, x = tr['all_h'][0], tr['all_x'][0]
    for l in range(synth.DEFAULT_MODEL_CONFIG['num_layers']):
        h, x = ref(l, h, x)
        assert torch.equal(h, tr['all_h'][l + 1]) and torch.equal(x, tr['all_x'][l + 1]), 'layer %d' % l
    lig = tr['mask_ligand']
    moved = not torch.equal(tr['all_x'][-1][lig], tr['all_x'][0][lig])
    assert moved == (cfgd.get('num_h2x', 1) > 0)


def test_sync_twoup_and_h2x_count_change_the_layer():
    """The float64 layer reads the form: sync_twoup and a second h2x change x, a second x2h changes h (guards against a reference that
    ignores the keys)."""
    base = {'num_x2h': 2, 'num_h2x': 2}
    sd = synth.make_state_dict(4, base, schedules=restate.make_schedules(base))
    b = synth.make_batch(2, 1, n_protein=50, ligand_sizes=[10])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    layer_forms.forward(sd, dict(base, num_layers=1), pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    h0, x0 = tr['all_h'][0], tr['all_x'][0]
    out = {}
    for name, c in (('base', base), ('sync', dict(base, sync_twoup=True)), ('one_h2x', dict(base, num_h2x=1)), ('one_x2h', dict(base, num_x2h=1))):
        out[name] = layer_forms.LayerFormRef.from_trace(sd, c, tr)(0, h0, x0)
    assert torch.equal(out['sync'][0], out['base'][0]) and not torch.equal(out['sync'][1], out['base'][1])
    assert torch.equal(out['one_h2x'][0], out['base'][0]) and not torch.equal(out['one_h2x'][1], out['base'][1])
    assert not torch.equal(out['one_x2h'][0], out['base'][0])


@pytest.mark.parametrize('cfgd', LAYER_FORM_CONFIGS + [{'num_x2h': 16, 'num_h2x': 16, 'num_layers': 1}], ids=option_id)
def test_model_state_dict_layout_matches_spec(cfgd):
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    c = default_model_config()
    c.update(cfgd)
    m = ScorePosNet3D(c, 27, 13)
    spec = synth.state_dict_spec(cfgd)
    sd = m.state_dict()
    assert list(sd.keys()) == [k for k, _, _ in spec]
    assert all(tuple(sd[k].shape) == tuple(s) for k, s, _ in spec)
    m.load_state_dict(synth.make_state_dict(0, cfgd, schedules=restate.make_schedules(cfgd)), strict=True)


def test_check_supported_rejects_out_of_range_forms():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    for bad in ({'num_x2h': 17}, {'num_h2x': -1}, {'num_h2x': 17}, {'sync_twoup': 'yes'}, {'num_x2h': 1.5}):
        c = default_model_config()
        c.update(bad)
        with pytest.raises(NotImplementedError):
            ScorePosNet3D(c, 27, 13)
    for ok in ({'num_x2h': 0}, {'num_h2x': 16}, {'sync_twoup': True}):
        c = default_model_config()
        c.update(ok)
        ScorePosNet3D(c, 27, 13)


def test_sublayer_code():
    from targetdiff_b200.score_model import sublayer_code
    assert sublayer_code({}) == 0
    assert sublayer_code({'num_x2h': 1, 'num_h2x': 1, 'sync_twoup': False}) == 0
    assert sublayer_code({'num_x2h': 2}) == 1 << 24 | 1 << 8 | 2
    assert sublayer_code({'num_x2h': 0, 'num_h2x': 3, 'sync_twoup': True}) == 1 << 24 | 1 << 16 | 3 << 8
    assert sublayer_code({'sync_twoup': True}) == 1 << 24 | 1 << 16 | 1 << 8 | 1


def test_tdiff_create_rejects_bad_sublayers():
    """tdiff_create validates the layer form before it looks for a device (TDIFF_EINVAL on any machine)."""
    from targetdiff_b200 import _lib
    lib = _lib.load()
    for code in (1, 0x7f, 2 << 24 | 0x0101, 1 << 24 | 17, 1 << 24 | 17 << 8, 1 << 24 | 2 << 16 | 0x0101, -1):
        cfg = _lib.tdiff_config(128, 16, 9, 32, 20, 13, 27, 1000, 0, 1, 0, 0, 0, 0, code)
        out = ctypes.c_void_p()
        rc = lib.tdiff_create(ctypes.byref(cfg), (_lib.tdiff_tensor * 1)(), 0, 0, ctypes.byref(out))
        assert rc == _lib.TDIFF_EINVAL and b'sublayers' in lib.tdiff_last_error(), hex(code)
    cfg = _lib.tdiff_config(128, 16, 9, 32, 20, 13, 27, 1000)
    cfg.reserved[0] = 1
    assert lib.tdiff_create(ctypes.byref(cfg), (_lib.tdiff_tensor * 1)(), 0, 0, ctypes.byref(ctypes.c_void_p())) == _lib.TDIFF_EINVAL


def test_ctypes_table_has_forward_blocks():
    from targetdiff_b200 import _lib
    assert 'tdiff_forward_blocks' in _lib.SIGNATURES
    assert hasattr(_lib.load(), 'tdiff_forward_blocks')
