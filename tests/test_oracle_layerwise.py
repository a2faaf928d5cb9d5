"""oracle/layerwise.py, the float64 one-layer reference of tests/test_gpu_layer_parity.py, checked against restate.forward (CPU only).

At fp32 it must be restate.forward's own layer, bit for bit; at float64 each layer must agree with the fp32 one to fp32 rounding."""
import pytest
import torch

from oracle import layerwise, restate, synth


def _trace(cfg, seed, n_protein, sizes):
    sd = synth.make_state_dict(seed, cfg, schedules=restate.make_schedules(cfg))
    b = synth.make_batch(seed + 5, len(sizes), n_protein=n_protein, ligand_sizes=sizes)
    pp, lp, _ = restate.center_pos(b['protein_pos'], b['init_ligand_pos'], b['batch_protein'], b['batch_ligand'])
    tr = {}
    restate.forward(sd, cfg, pp, b['protein_v'], b['batch_protein'], lp, b['init_ligand_v'], b['batch_ligand'], trace=tr)
    return sd, tr


CASES = [({}, 60, [9, 1, 14]), ({'cutoff_mode': 'hybrid', 'knn': 8}, 40, [7, 1, 12])]


@pytest.mark.parametrize('cfg,n_protein,sizes', CASES, ids=['knn32', 'hybrid8'])
def test_layerwise_fp32_chain_is_restate_forward(cfg, n_protein, sizes):
    sd, tr = _trace(cfg, 3, n_protein, sizes)
    ref = layerwise.LayerRef.from_trace(sd, cfg, tr, dtype=torch.float32)
    h, x = tr['all_h'][0], tr['all_x'][0]
    for l in range(synth.DEFAULT_MODEL_CONFIG['num_layers']):
        h, x = ref(l, h, x)
        assert h.dtype == torch.float32
        assert torch.equal(h, tr['all_h'][l + 1]) and torch.equal(x, tr['all_x'][l + 1]), 'layer %d' % l


@pytest.mark.parametrize('cfg,n_protein,sizes', CASES, ids=['knn32', 'hybrid8'])
def test_layerwise_fp64_agrees_with_fp32(cfg, n_protein, sizes):
    """Each layer in float64 on the fp32 chain's own input, relative to the layer's update (layerwise.row_error): the fp32 layer's
    h is within ~1e-6 of it; its ligand positions within a few 1e-5 (the update is ~1e-2 of the coordinates, so rounding x itself
    to fp32 is already ~1e-5 of the update; measured at most 1.4e-5)."""
    sd, tr = _trace(cfg, 3, n_protein, sizes)
    ref = layerwise.LayerRef.from_trace(sd, cfg, tr)
    assert torch.get_default_dtype() == torch.float32
    lig = tr['mask_ligand']
    for l in range(synth.DEFAULT_MODEL_CONFIG['num_layers']):
        h_in, x_in = tr['all_h'][l], tr['all_x'][l]
        h64, x64 = ref(l, h_in, x_in)
        assert h64.dtype == x64.dtype == torch.float64 and torch.get_default_dtype() == torch.float32
        eh = layerwise.row_error(tr['all_h'][l + 1], h64, h_in)
        ex = layerwise.row_error(tr['all_x'][l + 1], x64, x_in, lig)
        assert 0 < eh.max() < 2e-6 and 0 < ex.max() < 5e-5, (l, float(eh.max()), float(ex.max()))
        assert torch.equal(x64[~lig], x_in[~lig].double())          # protein atoms never move
