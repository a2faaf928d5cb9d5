"""Configuration surface of the sampling path (reference utils/misc.py:23-25, configs/training.yml, configs/sampling.yml)."""
import math
import numbers

import yaml


class Config(dict):
    """Attribute-access dict (what the reference gets from easydict.EasyDict; reference utils/misc.py:23-25)."""

    def __init__(self, d=None, **kw):
        super().__init__()
        for k, v in dict(d or {}, **kw).items():
            self[k] = v

    def __setitem__(self, k, v):
        if isinstance(v, dict) and not isinstance(v, Config):
            v = Config(v)
        super().__setitem__(k, v)

    __setattr__ = __setitem__

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def load_config(path):
    with open(path, 'r') as f:
        return Config(yaml.safe_load(f))


def default_model_config():
    """The `model:` section of the reference's configs/training.yml:9-42 (the checkpoint carries this config)."""
    return Config(
        model_mean_type='C0', beta_schedule='sigmoid', beta_start=1.e-7, beta_end=2.e-3, v_beta_schedule='cosine', v_beta_s=0.01,
        num_diffusion_timesteps=1000, loss_v_weight=100., sample_time_method='symmetric', time_emb_dim=0, time_emb_mode='simple',
        center_pos_mode='protein', node_indicator=True, model_type='uni_o2', num_blocks=1, num_layers=9, hidden_dim=128, n_heads=16,
        edge_feat_dim=4, num_r_gaussian=20, knn=32, num_node_types=8, act_fn='relu', norm=True, cutoff_mode='knn',
        ew_net_type='global', num_x2h=1, num_h2x=1, r_max=10., x2h_out_fc=False, sync_twoup=False)


def default_sampling_config():
    """reference configs/sampling.yml:1-10"""
    return Config(model=Config(checkpoint='./pretrained_models/pretrained_diffusion.pt'),
                  sample=Config(seed=2021, num_samples=100, num_steps=1000, pos_only=False, center_pos_mode='protein',
                                sample_num_atoms='prior'))


def sampling_time_seq(sample, T):
    """The time sequence `sample.respaced_steps` = n asks for (sampling.respaced_time_seq(T, n), an extension beyond the reference's
    sampling.yml), or None for the default chain.  ValueError when it is given with a `sample.num_steps` other than T: the two would
    ask for different chains."""
    n = sample.get('respaced_steps')
    if n is None:
        return None
    steps = sample.get('num_steps', T)
    if steps is not None and int(steps) != T:
        raise ValueError('sample.respaced_steps=%s cannot be combined with sample.num_steps=%s (num_steps truncates the chain; '
                         'leave it at T = %d)' % (n, steps, T))
    from .sampling import respaced_time_seq
    return respaced_time_seq(T, n)


def sampling_start(sample, T, start_ligand):
    """(start time t0, time sequence) of a chain from a start ligand (an extension beyond the reference's sampling.yml), or
    (None, None) without one (`start_ligand` False).  `sample.start_time` is required with a start ligand and refused without one;
    the sequence is t0, t0 - 1, ..., 0, or with `sample.respaced_steps` = n sampling.respaced_time_seq(T, n, start=t0).  ValueError
    with a `sample.num_steps` other than T, as for sampling_time_seq: the start time sets the chain's length."""
    t0 = sample.get('start_time')
    if not start_ligand:
        if t0 is not None:
            raise ValueError('sample.start_time=%s needs a start ligand (--start_ligand)' % (t0,))
        return None, None
    if t0 is None:
        raise ValueError('a start ligand (--start_ligand) needs sample.start_time in the config')
    t0 = int(t0)
    if not 0 <= t0 <= T - 1:
        raise ValueError('sample.start_time=%d outside 0..T-1 = %d' % (t0, T - 1))
    steps = sample.get('num_steps', T)
    if steps is not None and int(steps) != T:
        raise ValueError('sample.start_time=%d cannot be combined with sample.num_steps=%s (the start time sets the chain; '
                         'leave num_steps at T = %d)' % (t0, steps, T))
    n = sample.get('respaced_steps')
    if n is None:
        return t0, list(range(t0, -1, -1))
    from .sampling import respaced_time_seq
    return t0, respaced_time_seq(T, n, start=t0)


def check_resampling(sample, held):
    """(r, j) of `sample.resamplings` (default 1: no resampling) and `sample.jump_length` (default 1), an extension beyond the
    reference's sampling.yml.  ValueError unless both are integers >= 1, and for r > 1 when nothing is `held` (no fragment and no kept
    atoms): re-noising then only multiplies the cost."""
    r, j = sample.get('resamplings', 1), sample.get('jump_length', 1)
    for name, x in (('resamplings', r), ('jump_length', j)):
        if isinstance(x, bool) or not isinstance(x, int) or x < 1:
            raise ValueError('sample.%s must be an integer >= 1, got %r' % (name, x))
    if r > 1 and not held:
        raise ValueError('sample.resamplings=%d needs held atoms (--fragment, or kept atoms of a --start_ligand): without them '
                         'resampling only multiplies the cost' % r)
    return r, j


def check_clash_guidance(radius, strength):
    """(radius, strength) as floats, or ValueError unless they are a clash-guidance setting (DESIGN.md section 1): strength finite and
    >= 0, 0 turning guidance off (radius is then ignored and returned as None); with strength > 0 a finite radius > 0 in Angstrom.
    The same refusals as tdiff_set_clash_guidance.  ScorePosNet3D.sample_diffusion and the config keys (sample_clash_guidance) use it."""
    if isinstance(strength, bool) or not isinstance(strength, numbers.Real):
        raise ValueError('clash_strength must be a number, got %r' % (strength,))
    strength = float(strength)
    if not math.isfinite(strength) or strength < 0:
        raise ValueError('clash_strength must be finite and >= 0 (0 turns guidance off), got %r' % strength)
    if strength == 0:
        return None, 0.0
    if radius is None:
        raise ValueError('clash_strength=%g needs a clash_radius' % strength)
    if isinstance(radius, bool) or not isinstance(radius, numbers.Real) or not math.isfinite(float(radius)) or float(radius) <= 0:
        raise ValueError('clash_radius must be a finite number > 0 (Angstrom), got %r' % (radius,))
    return float(radius), strength


def sample_clash_guidance(sample):
    """(radius, strength) of `sample.clash_radius` and `sample.clash_strength` (an extension beyond the reference's sampling.yml):
    strength defaults to 0 (off) and the radius has no default.  check_clash_guidance's refusals, as ValueError."""
    return check_clash_guidance(sample.get('clash_radius'), sample.get('clash_strength', 0.0))


def sample_allowed_classes(sample, mode):
    """Sorted class indices of the ligand atom mode `mode` that the element constraint of `sample.allowed_elements` (element symbols,
    e.g. [C, N, O]: every class of those elements) or `sample.allowed_classes` (class indices) allows, or None without either (an
    extension beyond the reference's sampling.yml, DESIGN.md section 1).  ValueError when both are given, for an empty list, an
    unknown symbol (the message lists the mode's elements) or a class outside 0..K-1."""
    from .pocket import LIGAND_CLASS_ELEMENTS, element_classes
    el, cl = sample.get('allowed_elements'), sample.get('allowed_classes')
    if el is not None and cl is not None:
        raise ValueError('give sample.allowed_elements or sample.allowed_classes, not both')
    if el is None and cl is None:
        return None
    if el is not None:
        if isinstance(el, str) or not isinstance(el, (list, tuple)):
            raise ValueError('sample.allowed_elements must be a list of element symbols, got %r' % (el,))
        return element_classes(el, mode)
    K = len(LIGAND_CLASS_ELEMENTS[mode])
    if not isinstance(cl, (list, tuple)) or not cl:
        raise ValueError('sample.allowed_classes must be a non-empty list of class indices, got %r' % (cl,))
    for c in cl:
        if isinstance(c, bool) or not isinstance(c, int) or not 0 <= c < K:
            raise ValueError('sample.allowed_classes: %r is not a class index of the %s mode (0..%d)' % (c, mode, K - 1))
    return sorted(set(cl))


def check_connect_guidance(radius, length, strength):
    """(radius, length, strength) as floats, or ValueError unless they are a connectivity-guidance setting (DESIGN.md section 1):
    strength finite and >= 0, 0 turning guidance off (radius and length are then ignored and returned as None); with strength > 0 a
    finite bond radius > 0 and a bond length with 0 < length < radius, in Angstrom.  The same refusals as tdiff_set_connect_guidance.
    ScorePosNet3D.sample_diffusion and the config keys (sample_connect_guidance) use it."""
    if isinstance(strength, bool) or not isinstance(strength, numbers.Real):
        raise ValueError('connect_strength must be a number, got %r' % (strength,))
    strength = float(strength)
    if not math.isfinite(strength) or strength < 0:
        raise ValueError('connect_strength must be finite and >= 0 (0 turns guidance off), got %r' % strength)
    if strength == 0:
        return None, None, 0.0
    for name, x in (('connect_radius', radius), ('connect_length', length)):
        if x is None:
            raise ValueError('connect_strength=%g needs a %s' % (strength, name))
        if isinstance(x, bool) or not isinstance(x, numbers.Real) or not math.isfinite(float(x)) or float(x) <= 0:
            raise ValueError('%s must be a finite number > 0 (Angstrom), got %r' % (name, x))
    if not float(length) < float(radius):
        raise ValueError('connect_length=%g must be below connect_radius=%g' % (float(length), float(radius)))
    return float(radius), float(length), strength


def sample_connect_guidance(sample):
    """(radius, length, strength) of `sample.connect_radius`, `sample.connect_length` and `sample.connect_strength` (an extension
    beyond the reference's sampling.yml): strength defaults to 0 (off); radius and length have no default.  check_connect_guidance's
    refusals, as ValueError."""
    return check_connect_guidance(sample.get('connect_radius'), sample.get('connect_length'), sample.get('connect_strength', 0.0))


def sampling_time_path(sample, T, base, held):
    """The resampled time path of check_resampling's (r, j): sampling.resampled_time_path over `base`, the chain's decreasing time
    sequence (T - 1, ..., 0 when it is None), or None when r = 1."""
    r, j = check_resampling(sample, held)
    if r == 1:
        return None
    from .sampling import resampled_time_path
    return resampled_time_path(list(range(T - 1, -1, -1)) if base is None else base, r, j)


# Values the sm_90a engine implements; anything else is rejected loudly (SURVEY.md 8(b) "should-reject-clearly").
_SUPPORTED = dict(model_mean_type=('C0', 'noise'), beta_schedule=('sigmoid', 'linear', 'quad', 'const', 'jsd', 'cosine'),
                  v_beta_schedule=('cosine',), node_indicator=(True,), model_type=('uni_o2',),
                  hidden_dim=(128,), n_heads=(16,), edge_feat_dim=(4,), num_r_gaussian=(20,), act_fn=('relu',),
                  norm=(True,), cutoff_mode=('knn', 'hybrid'), ew_net_type=('global', 'r', 'm', 'none'),
                  num_x2h=tuple(range(17)), num_h2x=tuple(range(17)), x2h_out_fc=(False, True), sync_twoup=(False, True))
_WHY_NOT = {
    'cutoff_mode': "'radius' crashes in the reference itself (models/uni_transformer.py:278 reads an undefined self.r)",
    'model_type': "the EGNN backbone is outside the sampling path of the default model (SURVEY.md section 2)",
}


def check_supported(cfg):
    for k, allowed in _SUPPORTED.items():
        if k in cfg and cfg[k] not in allowed:
            raise NotImplementedError('config %s=%r is not implemented by the H100 engine (supported: %s)%s' % (
                k, cfg[k], list(allowed), '; ' + _WHY_NOT[k] if k in _WHY_NOT else ''))
    if not (1 <= int(cfg.knn) <= 64):
        raise NotImplementedError('knn=%r outside 1..64' % (cfg.knn,))
    if not (1 <= int(cfg.get('num_blocks', 1)) <= 16):
        raise NotImplementedError('num_blocks=%r outside 1..16' % (cfg.num_blocks,))
    if int(cfg.get('time_emb_dim', 0)) > 0 and cfg.get('time_emb_mode', 'simple') != 'simple':
        # 'sin' cannot run in the reference either: `time_feat` is [B, dim] but is concatenated with the [Nl, K] one-hot
        # (models/molopt_score_model.py:325-326)
        raise NotImplementedError("time_emb_mode=%r: only 'simple' is implemented (the reference's 'sin' branch fails on a shape mismatch)"
                                  % (cfg.time_emb_mode,))
