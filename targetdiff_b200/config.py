"""Configuration surface of the sampling path (reference utils/misc.py:23-25, configs/training.yml, configs/sampling.yml)."""
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


# Values the sm_90a engine implements; anything else is rejected loudly (SURVEY.md 8(b) "should-reject-clearly").
_SUPPORTED = dict(model_mean_type=('C0', 'noise'), beta_schedule=('sigmoid', 'linear', 'quad', 'const', 'jsd', 'cosine'),
                  v_beta_schedule=('cosine',), node_indicator=(True,), model_type=('uni_o2',),
                  hidden_dim=(128,), n_heads=(16,), edge_feat_dim=(4,), num_r_gaussian=(20,), act_fn=('relu',),
                  norm=(True,), cutoff_mode=('knn', 'hybrid'), ew_net_type=('global', 'r', 'm', 'none'), num_x2h=(1,), num_h2x=(1,),
                  x2h_out_fc=(False, True), sync_twoup=(False,))
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
