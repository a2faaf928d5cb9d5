"""Import the UNMODIFIED reference model from a reference checkout ($TARGETDIFF_REFERENCE) under the oracle shims.

Infrastructure for regenerating golden data (oracle/make_golden.py, oracle/make_reference_pins.py); nothing in the
test-suite, smoke() or bench.py calls it.
"""
import contextlib
import os
import sys

REFERENCE_ROOT = os.environ.get('TARGETDIFF_REFERENCE', '')
SHIMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'shims')


def reference_available():
    return os.path.isfile(os.path.join(REFERENCE_ROOT, 'models', 'molopt_score_model.py'))


def import_reference():
    """Returns the reference's `models.molopt_score_model` module (imported once)."""
    if not reference_available():
        raise RuntimeError('reference tree not present at %s' % REFERENCE_ROOT)
    for p in (SHIMS, REFERENCE_ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    import importlib
    return importlib.import_module('models.molopt_score_model')


def import_reference_scripts():
    """The reference's sampling drivers, UNMODIFIED: returns (scripts.sample_diffusion, scripts.sample_for_pocket).
    Needs, on top of the model shims, torch_geometric.data/transforms stand-ins and inert placeholders for the
    import-only dependencies rdkit / openbabel / lmdb (oracle/shims/_absent.py)."""
    import_reference()
    import importlib
    sys.path.insert(0, SHIMS) if SHIMS not in sys.path else None
    import _absent
    _absent.install()
    return importlib.import_module('scripts.sample_diffusion'), importlib.import_module('scripts.sample_for_pocket')


def default_model_config():
    """`configs/training.yml` model section (reference configs/training.yml:9-42) as an EasyDict."""
    import yaml
    sys.path.insert(0, SHIMS) if SHIMS not in sys.path else None
    from easydict import EasyDict
    with open(os.path.join(REFERENCE_ROOT, 'configs', 'training.yml')) as f:
        return EasyDict(yaml.safe_load(f)).model


@contextlib.contextmanager
def noise_tape(pos_noise, v_uniform):
    """Replace torch.randn_like / torch.rand_like by reads from a pre-drawn tape while the reference's
    `sample_diffusion` runs (draw order per step: randn_like(ligand_pos) then rand_like(log_model_prob),
    reference models/molopt_score_model.py:677-679,685 via :160-166)."""
    import torch
    state = {'p': 0, 'u': 0}
    orig_randn_like, orig_rand_like = torch.randn_like, torch.rand_like

    def randn_like(t, *a, **k):
        out = pos_noise[state['p']].to(t)
        assert out.shape == t.shape
        state['p'] += 1
        return out.clone()

    def rand_like(t, *a, **k):
        out = v_uniform[state['u']].to(t)
        assert out.shape == t.shape
        state['u'] += 1
        return out.clone()

    orig_normal_ = torch.Tensor.normal_

    def normal_(t, *a, **k):            # `pos_noise.normal_()` of likelihood_estimation (:581-582) reads the position tape too
        out = pos_noise[state['p']].to(t)
        assert out.shape == t.shape
        state['p'] += 1
        return t.copy_(out)

    torch.randn_like, torch.rand_like, torch.Tensor.normal_ = randn_like, rand_like, normal_
    try:
        yield state
    finally:
        torch.randn_like, torch.rand_like, torch.Tensor.normal_ = orig_randn_like, orig_rand_like, orig_normal_
