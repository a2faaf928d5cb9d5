"""Edge-MLP LayerNorm gains of either sign, and zero, against the oracle in every edge-MLP execution mode (run with -m gpu).

The engine packs every edge MLP reparameterised (engine.cu, pack_edge_mlp): the first Linear is centred over its 128 outputs, the sign
of each LayerNorm gain moves into the first Linear (default mode) or stays as a gain of +-1 (older modes), the gain's magnitude is
folded into the second Linear, and a feature whose gain is zero (or so small that bias / |gain| overflows) becomes a constant in the
output bias.  The synthetic weights of the other tests have gains 1 + 0.1 N(0, 1), all positive, so none of them reaches the sign or
the zero branch; here about half of every edge MLP's gains are negated, one is zero and one is subnormal."""
import pytest
import torch

from oracle import restate, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
EDGE_MLPS = ('.hk_func.', '.hv_func.', '.xk_func.', '.xv_func.')


def _signed_gain_state_dict(seed):
    sd = synth.make_state_dict(seed, schedules=restate.make_schedules())
    g = torch.Generator().manual_seed(seed + 1000)
    n = 0
    for key in list(sd):
        if key.endswith('.net.1.weight') and any(m in key for m in EDGE_MLPS):
            w, b = sd[key].clone(), sd[key[:-len('weight')] + 'bias'].clone()
            w[torch.rand(w.shape, generator=g) < 0.5] *= -1.0
            w[5], b[5] = 0.0, 0.3              # constant feature relu(0.3)
            w[77], b[77] = -1e-40, 0.2         # bias / |gain| overflows fp32: also a constant feature
            sd[key], sd[key[:-len('weight')] + 'bias'] = w, b
            n += 1
    assert n == 2 + 9 * 4                      # hk, hv of the (unused) init layer; hk, hv, xk, xv of the 9 layers
    return sd


@pytest.mark.parametrize('mode', ['simt', 'tc3v2', 'tc6', 'tc3'])
def test_signed_and_zero_ln_gains_vs_oracle(mode, monkeypatch):
    from targetdiff_b200 import _lib
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    monkeypatch.setenv('TDIFF_EDGE_MLP', mode)
    sd = _signed_gain_state_dict(1)
    model = ScorePosNet3D(default_model_config(), synth.PROTEIN_FEATURE_DIM, synth.LIGAND_NUM_CLASSES)
    model.load_state_dict(sd, strict=True)
    model = model.to(DEV)
    b = synth.make_batch(31, 3, n_protein=150, ligand_sizes=[20, 1, 33])
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    want = restate.forward(sd, None, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    out = model(pp.to(DEV), b['protein_v'].to(DEV), b['batch_protein'].to(DEV), lp.to(DEV), b['init_ligand_v'].to(DEV), b['batch_ligand'].to(DEV))
    assert _lib.load().tdiff_edge_mlp_mode(model.engine(DEV)) == {'simt': 0, 'tc3v2': 2, 'tc6': 3, 'tc3': 5}[mode]
    assert torch.equal(out['edge_index'].cpu(), tr['edge_index'])
    torch.testing.assert_close(out['pred_ligand_pos'].cpu(), want['pred_ligand_pos'], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out['pred_ligand_v'].cpu(), want['pred_ligand_v'], rtol=0, atol=1e-3)
    torch.testing.assert_close(out['final_h'].cpu(), want['final_h'], rtol=1e-4, atol=1e-4)
