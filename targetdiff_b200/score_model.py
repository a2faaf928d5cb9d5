"""ScorePosNet3D -- drop-in for the reference class of the same name on the sampling path.

Mirrors the reference's Python surface (models/molopt_score_model.py:200-368,633-703): constructor signature,
`state_dict` layout (all 384 entries of the default config, incl. the dead `refine_net.init_h_emb_layer.*` weights and the
15 schedule tables, so `load_state_dict(ckpt['model'])` is strict-compatible), `forward`, `sample_diffusion`, and the
module-level `log_sample_categorical` / `center_pos` helpers that scripts/sample_diffusion.py imports.

The modules below only *hold parameters*: every computation goes through libtdiff.so (hand-written sm_90a kernels,
include/tdiff.h).  There is no PyTorch/CPU execution path; calling forward on CPU tensors raises.
"""
import ctypes
import math

import numpy as np
import torch
import torch.nn.functional as F
import torch.nn as nn

from . import _lib
from .config import Config, check_clash_guidance, check_connect_guidance, check_supported

GAUSSIAN_OFFSETS = (0, 1, 1.25, 1.5, 1.75, 2, 2.25, 2.5, 2.75, 3, 3.5, 4, 4.5, 5, 5.5, 6, 7, 8, 9, 10)   # models/common.py:15


# ----------------------------------------------------------------------------------------------------------------
# noise schedules (fp64 numpy -> fp32 tables; semantics of models/molopt_score_model.py:48-97,169-170,221-267)
# ----------------------------------------------------------------------------------------------------------------
def position_betas(kind, beta_start, beta_end, T):
    if kind == 'sigmoid':
        grid = np.linspace(-6, 6, T)
        return (1 / (np.exp(-grid) + 1)) * (beta_end - beta_start) + beta_start
    if kind == 'linear':
        return np.linspace(beta_start, beta_end, T, dtype=np.float64)
    if kind == 'quad':
        return np.linspace(beta_start ** 0.5, beta_end ** 0.5, T, dtype=np.float64) ** 2
    if kind == 'const':
        return beta_end * np.ones(T, dtype=np.float64)
    if kind == 'jsd':
        return 1.0 / np.linspace(T, 1, T, dtype=np.float64)
    raise NotImplementedError(kind)


def cosine_alpha_sqrt(T, s):
    grid = np.linspace(0, T + 1, T + 1)
    cum = np.cos(((grid / (T + 1)) + s) / (1 + s) * np.pi * 0.5) ** 2
    cum = cum / cum[0]
    return np.sqrt(np.clip(cum[1:] / cum[:-1], a_min=0.001, a_max=1.))


def diffusion_tables(cfg):
    """name -> fp32 tensor for the 15 schedule entries of the state_dict."""
    T = int(cfg.num_diffusion_timesteps)
    if cfg.beta_schedule == 'cosine':
        alphas = cosine_alpha_sqrt(T, cfg.pos_beta_s) ** 2
        betas = 1. - alphas
    else:
        betas = position_betas(cfg.beta_schedule, cfg.beta_start, cfg.beta_end, T)
        alphas = 1. - betas
    cum = np.cumprod(alphas, axis=0)
    cum_prev = np.append(1., cum[:-1])
    t32 = lambda a: torch.from_numpy(np.asarray(a)).float()
    tab = dict(
        betas=t32(betas), alphas_cumprod=t32(cum), alphas_cumprod_prev=t32(cum_prev), sqrt_alphas_cumprod=t32(np.sqrt(cum)),
        sqrt_one_minus_alphas_cumprod=t32(np.sqrt(1. - cum)), sqrt_recip_alphas_cumprod=t32(np.sqrt(1. / cum)),
        sqrt_recipm1_alphas_cumprod=t32(np.sqrt(1. / cum - 1)),
        posterior_mean_c0_coef=t32(betas * np.sqrt(cum_prev) / (1. - cum)),
        posterior_mean_ct_coef=t32((1. - cum_prev) * np.sqrt(alphas) / (1. - cum)))
    var32 = t32(betas * (1. - cum_prev) / (1. - cum))
    tab['posterior_var'] = var32
    # entry 0 of the variance is 0 -> the log table repeats entry 1 there (taken from the fp32 table, like the reference)
    tab['posterior_logvar'] = t32(np.log(np.append(var32[1], var32[1:])))
    if cfg.v_beta_schedule != 'cosine':
        raise NotImplementedError(cfg.v_beta_schedule)
    log_a = np.log(cosine_alpha_sqrt(T, cfg.v_beta_s))
    log_cum = np.cumsum(log_a)
    one_minus = lambda a: np.log(1 - np.exp(a) + 1e-40)
    tab.update(log_alphas_v=t32(log_a), log_one_minus_alphas_v=t32(one_minus(log_a)), log_alphas_cumprod_v=t32(log_cum),
               log_one_minus_alphas_cumprod_v=t32(one_minus(log_cum)))
    return tab


SCHEDULE_NAMES = ('betas', 'alphas_cumprod', 'alphas_cumprod_prev', 'sqrt_alphas_cumprod', 'sqrt_one_minus_alphas_cumprod',
                  'sqrt_recip_alphas_cumprod', 'sqrt_recipm1_alphas_cumprod', 'posterior_mean_c0_coef', 'posterior_mean_ct_coef',
                  'posterior_var', 'posterior_logvar', 'log_alphas_v', 'log_one_minus_alphas_v', 'log_alphas_cumprod_v',
                  'log_one_minus_alphas_cumprod_v')


# ----------------------------------------------------------------------------------------------------------------
# parameter containers (names chosen so that state_dict keys equal the reference's; SURVEY.md Appendix D)
# ----------------------------------------------------------------------------------------------------------------
class _Act(nn.Module):
    pass


class MLP(nn.Module):
    """Linear -> LayerNorm -> act -> Linear parameter holder (`net.0`, `net.1`, `net.3`; models/common.py:60-80)."""

    def __init__(self, in_dim, out_dim, hidden_dim):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(in_dim, hidden_dim), nn.LayerNorm(hidden_dim), _Act(), nn.Linear(hidden_dim, out_dim))


class _Offsets(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer('offset', torch.tensor(GAUSSIAN_OFFSETS, dtype=torch.float32))


class _X2H(nn.Module):
    """parameter holder of BaseX2HAttLayer (reference models/uni_transformer.py:11-40; same module order = same state_dict order)"""

    def __init__(self, H, kv_dim, r_dim, ew_net_type, out_fc):
        super().__init__()
        self.hk_func, self.hv_func, self.hq_func = MLP(kv_dim, H, H), MLP(kv_dim, H, H), MLP(H, H, H)
        if ew_net_type == 'r':
            self.ew_net = nn.Sequential(nn.Linear(r_dim, 1), _Act())
        elif ew_net_type == 'm':
            self.ew_net = nn.Sequential(nn.Linear(H, 1), _Act())
        if out_fc:
            self.node_output = MLP(2 * H, H, H)


class _H2X(nn.Module):
    """parameter holder of BaseH2XAttLayer (reference models/uni_transformer.py:86-106)"""

    def __init__(self, H, kv_dim, n_heads, r_dim, ew_net_type):
        super().__init__()
        self.xk_func, self.xv_func, self.xq_func = MLP(kv_dim, H, H), MLP(kv_dim, n_heads, H), MLP(H, H, H)
        if ew_net_type == 'r':
            self.ew_net = nn.Sequential(nn.Linear(r_dim, 1), _Act())


class _AttLayer(nn.Module):
    def __init__(self, H, n_heads, kv_dim, r_dim, num_x2h, num_h2x, ew_net_type, out_fc):
        super().__init__()
        self.distance_expansion = _Offsets()
        self.x2h_layers = nn.ModuleList([_X2H(H, kv_dim, r_dim, ew_net_type, out_fc) for _ in range(num_x2h)])
        self.h2x_layers = nn.ModuleList([_H2X(H, kv_dim, n_heads, r_dim, ew_net_type) for _ in range(num_h2x)])


class _RefineNet(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        H = cfg.hidden_dim
        r_dim = 4 * cfg.num_r_gaussian
        kv_dim = 2 * H + cfg.edge_feat_dim + r_dim
        ew, fc = cfg.ew_net_type, bool(cfg.x2h_out_fc)
        self.distance_expansion = _Offsets()
        if ew == 'global':
            self.edge_pred_layer = MLP(cfg.num_r_gaussian, 1, H)
        self.init_h_emb_layer = _AttLayer(H, cfg.n_heads, kv_dim, r_dim, 1, 0, ew, fc)      # never evaluated; present for strict loading
        self.base_block = nn.ModuleList([_AttLayer(H, cfg.n_heads, kv_dim, r_dim, cfg.num_x2h, cfg.num_h2x, ew, fc)
                                         for _ in range(cfg.num_layers)])


def log_sample_categorical(logits):
    """Gumbel-max sample of class indices (reference models/molopt_score_model.py:160-166); used for the initial
    ligand types by sample_diffusion_ligand.  Plain torch on whatever device `logits` lives on (plumbing, not hot path)."""
    uniform = torch.rand_like(logits)
    gumbel = -torch.log(-torch.log(uniform + 1e-30) + 1e-30)
    return (gumbel + logits).argmax(dim=-1)


def sublayer_code(cfg):
    """`tdiff_config.sublayers` for the layer form (num_x2h, num_h2x, sync_twoup): 0 for the reference default (1, 1, False)."""
    nx, nh, sync = int(cfg.get('num_x2h', 1)), int(cfg.get('num_h2x', 1)), int(bool(cfg.get('sync_twoup', False)))
    if (nx, nh, sync) == (1, 1, 0):
        return 0
    return 1 << 24 | sync << 16 | nh << 8 | nx


def check_time_seq(time_seq, T, start=None):
    """`time_seq` as a list of ints, or ValueError unless it is tau_0 > tau_1 > ... > tau_{S-1} >= 0 with tau_0 = T - 1, 1 <= S <= T;
    with a start time `start` (a chain from a start ligand, DESIGN.md section 1), tau_0 = start instead, in 0..T-1."""
    seq = [int(x) for x in (time_seq.tolist() if hasattr(time_seq, 'tolist') else time_seq)]
    if not seq:
        raise ValueError('time_seq is empty')
    if len(seq) > T:
        raise ValueError('time_seq has %d steps, more than T = %d' % (len(seq), T))
    if start is None:
        if seq[0] != T - 1:
            raise ValueError('time_seq must start at T - 1 = %d, not %d' % (T - 1, seq[0]))
    else:
        if not 0 <= int(start) <= T - 1:
            raise ValueError('start time %d outside 0..T-1 = %d' % (int(start), T - 1))
        if seq[0] != int(start):
            raise ValueError('time_seq must start at the start time %d, not %d' % (int(start), seq[0]))
    if any(b >= a for a, b in zip(seq, seq[1:])):
        raise ValueError('time_seq must be strictly decreasing')
    if seq[-1] < 0:
        raise ValueError('time_seq has a negative time %d' % seq[-1])
    return seq


PATH_MAX_PER_T = 64          # TDIFF_PATH_MAX_PER_T (include/tdiff.h): a time path has at most 64 T steps


def check_time_path(time_path, T, start=None):
    """`time_path` as a list of ints, or ValueError unless it is a time path (DESIGN.md section 1): every tau_s in 0..T-1, tau_0 = T - 1
    (the start time `start` with a start ligand), tau_{s+1} != tau_s, tau_1 < tau_0 when S > 1 (the first step evaluates the network),
    1 <= S <= PATH_MAX_PER_T * T."""
    path = [int(x) for x in (time_path.tolist() if hasattr(time_path, 'tolist') else time_path)]
    if not path:
        raise ValueError('time_path is empty')
    if len(path) > PATH_MAX_PER_T * T:
        raise ValueError('time_path has %d steps, more than %d T = %d' % (len(path), PATH_MAX_PER_T, PATH_MAX_PER_T * T))
    if start is None:
        if path[0] != T - 1:
            raise ValueError('time_path must start at T - 1 = %d, not %d' % (T - 1, path[0]))
    else:
        if not 0 <= int(start) <= T - 1:
            raise ValueError('start time %d outside 0..T-1 = %d' % (int(start), T - 1))
        if path[0] != int(start):
            raise ValueError('time_path must start at the start time %d, not %d' % (int(start), path[0]))
    bad = [x for x in path if not 0 <= x <= T - 1]
    if bad:
        raise ValueError('time_path has a time %d outside 0..T-1 = %d' % (bad[0], T - 1))
    for s, (a, b) in enumerate(zip(path, path[1:])):
        if a == b:
            raise ValueError('time_path repeats time %d at steps %d and %d' % (a, s, s + 1))
    if len(path) > 1 and path[1] > path[0]:
        raise ValueError('time_path goes up at its first step (%d -> %d); the first step must evaluate the network' % (path[0], path[1]))
    return path


def _counts_from_batch(batch, name):
    """Per-graph atom counts from a sorted PyG-style batch vector (host list)."""
    if batch.numel() == 0:
        return []
    if batch.numel() > 1 and bool((batch[1:] < batch[:-1]).any()):
        raise ValueError('%s must be sorted ascending (it is in the reference pipeline: Batch.from_data_list / repeat_interleave)' % name)
    return torch.bincount(batch).cpu().tolist()


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class ScorePosNet3D(nn.Module):

    def __init__(self, config, protein_atom_feature_dim, ligand_atom_feature_dim):
        super().__init__()
        if not isinstance(config, Config):
            config = Config(dict(config))
        check_supported(config)
        self.config = config
        self.model_mean_type = config.model_mean_type
        self.loss_v_weight = config.get('loss_v_weight', 100.)
        self.sample_time_method = config.get('sample_time_method', 'symmetric')
        for name, tab in diffusion_tables(config).items():
            setattr(self, name, nn.Parameter(tab, requires_grad=False))
        self.num_timesteps = self.betas.size(0)
        self.register_buffer('Lt_history', torch.zeros(self.num_timesteps))
        self.register_buffer('Lt_count', torch.zeros(self.num_timesteps))
        self.hidden_dim = config.hidden_dim
        self.num_classes = ligand_atom_feature_dim
        self.protein_atom_feature_dim = protein_atom_feature_dim
        emb_dim = self.hidden_dim - 1      # node_indicator=True
        self.protein_atom_emb = nn.Linear(protein_atom_feature_dim, emb_dim)
        self.center_pos_mode = config.center_pos_mode
        self.time_emb_dim = config.time_emb_dim
        self.time_emb_mode = config.time_emb_mode
        # time_emb_mode 'simple' appends time_step / T to the ligand one-hot (reference :289-291,319-324)
        self.ligand_atom_emb = nn.Linear(ligand_atom_feature_dim + (1 if self.time_emb_dim > 0 else 0), emb_dim)
        self.refine_net_type = config.model_type
        self.refine_net = _RefineNet(config)
        self.v_inference = nn.Sequential(nn.Linear(self.hidden_dim, self.hidden_dim), _Act(), nn.Linear(self.hidden_dim, ligand_atom_feature_dim))
        self.requires_grad_(False)          # inference engine: the CUDA path has no backward
        self._engine = None
        self._engine_device = None
        self._bound_key = None

    # ------------------------------------------------------------------ engine management
    def _apply(self, fn, *a, **k):
        self._drop_engine()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._drop_engine()
        return super().load_state_dict(*a, **k)

    def _drop_engine(self):
        eng = self.__dict__.get('_engine')
        if eng is not None:
            _lib.load().tdiff_destroy(eng)
        self.__dict__['_engine'] = None
        self.__dict__['_bound_key'] = None

    def __del__(self):
        try:
            self._drop_engine()
        except Exception:
            pass

    def engine(self, device):
        """The libtdiff engine for `device` (created on first use from the current state_dict)."""
        device = torch.device(device)
        if device.type != 'cuda':
            raise RuntimeError('ScorePosNet3D (targetdiff_b200) only runs on CUDA devices; got %s. There is no CPU path.' % device)
        index = device.index if device.index is not None else torch.cuda.current_device()
        if self._engine is not None and self._engine_device == index:
            return self._engine
        self._drop_engine()
        lib = _lib.load()
        sd = {k: v.detach().to('cpu', torch.float32).contiguous() for k, v in self.state_dict().items()}
        entries = (_lib.tdiff_tensor * len(sd))()
        keep = []
        for i, (k, v) in enumerate(sd.items()):
            name = k.encode()
            keep.append((name, v))
            entries[i].name, entries[i].data, entries[i].numel = name, v.data_ptr(), v.numel()
        cfg = _lib.tdiff_config(self.hidden_dim, self.config.n_heads, self.config.num_layers, self.config.knn, self.config.num_r_gaussian,
                                self.num_classes, self.protein_atom_feature_dim, self.num_timesteps,
                                {'C0': 0, 'noise': 1}[self.model_mean_type], int(self.config.num_blocks),
                                {'global': 0, 'r': 1, 'm': 2, 'none': 3}[self.config.ew_net_type], int(bool(self.config.x2h_out_fc)),
                                1 if self.time_emb_dim > 0 else 0, {'knn': 0, 'hybrid': 1}[self.config.get('cutoff_mode', 'knn')],
                                sublayer_code(self.config))
        out = ctypes.c_void_p()
        _lib.check(lib.tdiff_create(ctypes.byref(cfg), entries, len(sd), index, ctypes.byref(out)))
        self._engine, self._engine_device, self._bound_key = out, index, None
        return out

    @staticmethod
    def _stream(device):
        return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)

    def _bind(self, eng, protein_pos, protein_v, batch_protein, batch_ligand, center_mode):
        lib = _lib.load()
        pc = _counts_from_batch(batch_protein, 'batch_protein')
        lc = _counts_from_batch(batch_ligand, 'batch_ligand')
        B = max(len(pc), len(lc))
        pc += [0] * (B - len(pc))
        lc += [0] * (B - len(lc))
        if sum(pc) != protein_pos.shape[0] or protein_v.shape[0] != protein_pos.shape[0]:
            raise ValueError('protein arrays disagree with batch_protein')
        ppos = protein_pos.detach().to(torch.float32).contiguous()
        pfeat = protein_v.detach().to(torch.float32).contiguous()
        if pfeat.dim() != 2 or pfeat.shape[1] != self.protein_atom_feature_dim:
            raise ValueError('protein_v must be [Np,%d]' % self.protein_atom_feature_dim)
        _lib.check(lib.tdiff_bind_batch(eng, B, _lib.i32_array(pc), _lib.i32_array(lc), _ptr(ppos), _ptr(pfeat), center_mode,
                                        self._stream(ppos.device)))
        return B, sum(pc), sum(lc)

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    def forward(self, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand,
                time_step=None, return_all=False, fix_x=False, return_edge_weight=False):
        """One network evaluation (reference models/molopt_score_model.py:313-368; `time_step` [B] is only read with time_emb_dim > 0).
        Returns {'pred_ligand_pos','pred_ligand_v','final_h','final_ligand_h'}; additionally 'edge_index' (int64 [2,E]) and, with
        `return_edge_weight`, 'edge_weight' [E]: the global edge gate e_w in edge_index order (models/uni_transformer.py:312-316).
        `return_all` adds the reference's per-block lists (:360-367) of num_blocks + 1 tensors each: 'layer_pred_ligand_pos' (ligand
        coordinates before block 0 and after every block) and 'layer_pred_ligand_v' (the type head on the ligand features there)."""
        dev = protein_pos.device
        eng = self.engine(dev)
        lib = _lib.load()
        st = self._stream(dev)
        B, Np, Nl = self._bind(eng, protein_pos, protein_v, batch_protein, batch_ligand, 0)
        lpos = init_ligand_pos.detach().to(torch.float32).contiguous()
        lv = init_ligand_v.detach().to(torch.int64).contiguous()
        if lpos.shape[0] != Nl or lv.shape[0] != Nl:
            raise ValueError('ligand arrays disagree with batch_ligand')
        _lib.check(lib.tdiff_set_ligand(eng, _ptr(lpos), _ptr(lv), 0, st))
        if self.time_emb_dim > 0:           # (time_step / T) per graph, fp32 like the reference's true division (:322)
            if time_step is None:
                raise ValueError('time_step is required when time_emb_dim > 0')
            # divided by a tensor, not a Python number: torch's CUDA division by a scalar multiplies by the rounded reciprocal, which
            # is one ulp off the correctly rounded t / T for some t (9, 13, 18 of T = 20); the sampling chain's set_time_kernel and
            # the CPU oracle divide
            tn = time_step.to(dev, torch.float32)
            tn = (tn / torch.full_like(tn, float(self.num_timesteps))).contiguous()
            if tn.numel() != B:
                raise ValueError('time_step must have one entry per graph')
            _lib.check(lib.tdiff_set_time(eng, _ptr(tn), st))
        pred_pos = torch.empty(Nl, 3, device=dev)
        logits = torch.empty(Nl, self.num_classes, device=dev)
        final_h = torch.empty(Np + Nl, self.hidden_dim, device=dev)
        if return_all:
            nb = int(self.config.get('num_blocks', 1)) + 1
            block_pos = torch.empty(nb, Nl, 3, device=dev)
            block_logits = torch.empty(nb, Nl, self.num_classes, device=dev)
            _lib.check(lib.tdiff_forward_blocks(eng, _ptr(pred_pos), _ptr(logits), _ptr(final_h), int(bool(fix_x)), _ptr(block_pos),
                                                _ptr(block_logits), st))
        else:
            _lib.check(lib.tdiff_forward(eng, _ptr(pred_pos), _ptr(logits), _ptr(final_h), int(bool(fix_x)), st))
        E = lib.tdiff_num_edges(eng, st)
        if E < 0:
            _lib.check(int(E))
        edge_index = torch.empty(2, E, dtype=torch.int64, device=dev)
        _lib.check(lib.tdiff_get_edge_index(eng, _ptr(edge_index), st))
        # ligand rows of the composed node order: per graph, protein atoms then ligand atoms
        lig_rows = self._ligand_rows(batch_protein, batch_ligand, B, dev)
        out = {'pred_ligand_pos': pred_pos, 'pred_ligand_v': logits, 'final_h': final_h, 'final_ligand_h': final_h[lig_rows],
               'edge_index': edge_index}
        if return_all:
            out['layer_pred_ligand_pos'] = list(block_pos.unbind(0))
            out['layer_pred_ligand_v'] = list(block_logits.unbind(0))
        if return_edge_weight:
            e_w = torch.empty(E, device=dev)
            _lib.check(lib.tdiff_get_edge_weight(eng, _ptr(e_w), st))
            out['edge_weight'] = e_w
        return out

    @staticmethod
    def _ligand_rows(batch_protein, batch_ligand, B, dev):
        pc = torch.bincount(batch_protein, minlength=B)
        lc = torch.bincount(batch_ligand, minlength=B)
        lig_start = torch.cumsum(pc + lc, 0) - lc                 # node index of the first ligand atom of each graph
        first = torch.cumsum(lc, 0) - lc
        a = torch.arange(batch_ligand.numel(), device=dev)
        return lig_start[batch_ligand] + (a - first[batch_ligand])

    @torch.no_grad()
    def sample_diffusion(self, protein_pos, protein_v, batch_protein, init_ligand_pos, init_ligand_v, batch_ligand,
                         num_steps=None, center_pos_mode=None, pos_only=False, noise_tape=None, seed=None, return_traj=True,
                         stack_traj=False, fixed_mask=None, fixed_noise_tape=None, time_seq=None, start_time=None, start_noise_tape=None,
                         time_path=None, clash_radius=None, clash_strength=0.0, allowed_types=None, connect_radius=None,
                         connect_length=None, connect_strength=0.0):
        """The reverse-diffusion chain (reference models/molopt_score_model.py:633-703), executed entirely by libtdiff.so.

        Extensions over the reference signature (all optional): `noise_tape=(pos_noise [S,Nl,3], v_uniform [S,Nl,K])`
        replaces the RNG in the reference's draw order (parity tests); `seed` keys the device Philox generator (default:
        drawn from torch's global CPU generator, so `seed_all` makes runs reproducible); `return_traj=False` skips the
        four trajectory outputs; `stack_traj=True` returns each trajectory as one stacked CPU tensor [S, ...] instead
        of the reference's list of per-step tensors.

        Fixed atoms (fragment-conditioned sampling, DESIGN.md section 1): `fixed_mask` [Nl] bool holds the masked ligand atoms to the
        forward process of their `init_ligand_pos` / `init_ligand_v` rows (lab frame) through the chain; they end exactly there.
        `fixed_noise_tape=(pos_noise [S+1,Nl,3], v_uniform [S+1,Nl,K])` replaces their draws; it is required with `noise_tape` and
        not allowed without it.  pos_traj / v_traj show the fixed rows as held, v0_traj / vt_traj what the network made of them.

        Respaced sampling (DESIGN.md section 1): `time_seq` = tau_0 > ... > tau_{S-1} >= 0 with tau_0 = T - 1 runs S steps; step s
        evaluates the network at tau_s and moves the state to tau_{s+1} (to tau_{S-1} - 1 at the last step) with the exact jump
        posteriors.  `num_steps`, if given, must be S; tapes are [S, ...] (fixed tape [S+1, ...]) and trajectories [S, ...].
        `sampling.respaced_time_seq(T, n)` makes an evenly spaced one.  Sample quality at fewer steps is not measured.

        Start-ligand sampling (DESIGN.md section 1): with `start_time` = t0 in 0..T-1, `init_ligand_pos` / `init_ligand_v` are a clean
        start ligand; before the first step every row that is not fixed is replaced by a sample of q(x_t0 | x0), q(v_t0 | v0) (the types
        are kept with pos_only), fixed rows get their sample at t0, and the chain runs from t0: `time_seq` defaults to t0, t0 - 1, ..., 0
        (t0 + 1 steps) and must begin at t0.  `start_noise_tape=(pos_noise [Nl,3], v_uniform [Nl,K])` replaces the start draw (v_uniform
        may be None with pos_only); it is required with `noise_tape` and not allowed without it.  Sample quality is not measured.

        Resampled sampling (DESIGN.md section 1): `time_path` (check_time_path; e.g. sampling.resampled_time_path) runs a path whose
        steps may go up: step s moves the state from tau_s to p = tau_{s+1} (tau_{S-1} - 1 at the last step); a denoising step (p < tau_s)
        is time_seq's step, a re-noising step (p > tau_s) draws the state from the forward process q(x_p | x_t), q(v_p | v_t) without the
        network, and fixed rows are resampled at p after either.  Not with `time_seq`; it begins at the start time with `start_time`.
        Tapes are [S, ...] (fixed tape [S+1, ...]), trajectories [S, ...]; after a re-noising step v0_traj repeats the entry before and
        vt_traj holds the normalised log q(v_p | v_t).  Sample quality is not measured.

        Clash guidance (DESIGN.md section 1): with `clash_strength` = lambda > 0 and `clash_radius` = rho, every denoising step moves
        each ligand atom's x0 prediction y to y + lambda * sum (rho - d) (y - x_p) / d over the protein atoms x_p of its pocket at a
        distance 0 < d < rho before the posterior step.  Every call sets the engine's guidance, off included, so a call never inherits
        an earlier call's setting.  No random numbers are drawn.  Whether it improves molecules is not measured.

        Element constraints (DESIGN.md section 1): `allowed_types` [Nl, K] bool, row a the classes ligand atom a may end in (none
        empty).  Every denoising step conditions the type prediction on the allowed set (log v0_hat = -inf elsewhere) and the decoder
        step (the last step of a chain that ends at t = 0) draws from the posterior renormalised over it, so every atom of a chain
        that ends at t = 0 ends in an allowed class; intermediate states, and the last state of a chain that stops before t = 0, are
        not restricted.  Fixed rows are held as without it (give them every class).  v0_traj / vt_traj hold -inf at forbidden
        entries where those are their values.  Not with pos_only.  Every call sets or clears the engine's mask.  No random numbers
        are drawn.  Whether constrained molecules are chemically sensible is not measured.

        Connectivity guidance (DESIGN.md section 1): with `connect_strength` = lambda > 0, `connect_radius` = rho and `connect_length`
        = b (0 < b < rho), every denoising step, after clash guidance, pulls the separate pieces of each graph's predicted ligand
        together: atoms closer than rho are bonded (fixed rows at their targets), and each component without a fixed row moves rigidly
        by lambda * w * (d - b) along its closest outside pair (d its length; w = 1 towards a component with a fixed row, 1/2
        otherwise).  A graph in one piece keeps its prediction bit for bit.  At most 1024 ligand atoms per graph while it is on.  Every
        call sets the engine's setting, off included.  No random numbers are drawn.  Whether it improves molecules is not measured."""
        T = self.num_timesteps
        clash_radius, clash_strength = check_clash_guidance(clash_radius, clash_strength)
        connect_radius, connect_length, connect_strength = check_connect_guidance(connect_radius, connect_length, connect_strength)
        if allowed_types is not None and pos_only:
            raise ValueError('allowed_types constrains atom types, which pos_only=True keeps as they are')
        if time_path is not None:
            if time_seq is not None:
                raise ValueError('time_path cannot be combined with time_seq')
            time_path = check_time_path(time_path, T, start=start_time)
            if num_steps is not None and int(num_steps) != len(time_path):
                raise ValueError('num_steps=%d disagrees with a time_path of %d steps' % (int(num_steps), len(time_path)))
            num_steps = len(time_path)
        if start_time is not None:
            t0 = int(start_time)
            if not 0 <= t0 <= T - 1:
                raise ValueError('start_time %d outside 0..T-1 = %d' % (t0, T - 1))
            if time_seq is None and time_path is None:
                time_seq = list(range(t0, -1, -1))
            if (start_noise_tape is None) != (noise_tape is None):
                raise ValueError('start_noise_tape is required with noise_tape, and not allowed without it')
        elif start_noise_tape is not None:
            raise ValueError('start_noise_tape without start_time')
        if time_seq is not None:
            time_seq = check_time_seq(time_seq, T, start=start_time)
            if num_steps is not None and int(num_steps) != len(time_seq):
                raise ValueError('num_steps=%d disagrees with a time_seq of %d steps' % (int(num_steps), len(time_seq)))
            num_steps = len(time_seq)
        if num_steps is None:
            num_steps = self.num_timesteps
        mode = {None: 0, 'none': 0, 'protein': 1}.get(center_pos_mode, None)
        if mode is None:
            raise NotImplementedError(center_pos_mode)
        dev = protein_pos.device
        eng = self.engine(dev)
        lib = _lib.load()
        st = self._stream(dev)
        _lib.check(lib.tdiff_set_clash_guidance(eng, ctypes.c_float(clash_radius or 0.0), ctypes.c_float(clash_strength)))
        _lib.check(lib.tdiff_set_connect_guidance(eng, ctypes.c_float(connect_radius or 0.0), ctypes.c_float(connect_length or 0.0),
                                                  ctypes.c_float(connect_strength)))
        B, Np, Nl = self._bind(eng, protein_pos, protein_v, batch_protein, batch_ligand, mode)
        lpos = init_ligand_pos.detach().to(torch.float32).contiguous()
        lv = init_ligand_v.detach().to(torch.int64).contiguous()
        _lib.check(lib.tdiff_set_ligand(eng, _ptr(lpos), _ptr(lv), mode, st))
        S, K = int(num_steps), self.num_classes
        bits = None
        if allowed_types is not None:
            am = torch.as_tensor(allowed_types).detach().to(dev)
            if am.dtype != torch.bool or tuple(am.shape) != (Nl, K):
                raise ValueError('allowed_types must be a [Nl, K] = %s bool tensor, got %s %s' % ((Nl, K), tuple(am.shape), am.dtype))
            bits = (am.to(torch.int32) << torch.arange(K, dtype=torch.int32, device=dev)).sum(1, dtype=torch.int32).contiguous()
        _lib.check(lib.tdiff_set_type_mask(eng, _ptr(bits), st))                # None clears: a call never inherits a mask
        pos_noise = v_uniform = None
        if noise_tape is not None:
            pos_noise = noise_tape[0].detach().to(dev, torch.float32).contiguous()
            v_uniform = noise_tape[1].detach().to(dev, torch.float32).contiguous()
            if tuple(pos_noise.shape) != (S, Nl, 3) or tuple(v_uniform.shape) != (S, Nl, K):
                raise ValueError('noise tape shapes must be [S,Nl,3] and [S,Nl,K]')
        fix_pn = fix_vu = None
        if fixed_mask is not None:
            mask = torch.as_tensor(fixed_mask).detach().to(dev, torch.uint8).contiguous()
            if tuple(mask.shape) != (Nl,):
                raise ValueError('fixed_mask must have one entry per ligand atom: shape %s, %d atoms' % (tuple(mask.shape), Nl))
            if fixed_noise_tape is not None:
                fix_pn = fixed_noise_tape[0].detach().to(dev, torch.float32).contiguous()
                if tuple(fix_pn.shape) != (S + 1, Nl, 3):
                    raise ValueError('fixed noise tape positions must be [S+1,Nl,3] = %s, got %s' % ((S + 1, Nl, 3), tuple(fix_pn.shape)))
                if not pos_only:
                    fix_vu = fixed_noise_tape[1].detach().to(dev, torch.float32).contiguous()
                    if tuple(fix_vu.shape) != (S + 1, Nl, K):
                        raise ValueError('fixed noise tape uniforms must be [S+1,Nl,K] = %s, got %s' % ((S + 1, Nl, K), tuple(fix_vu.shape)))
            _lib.check(lib.tdiff_set_fixed(eng, _ptr(mask), _ptr(lpos), _ptr(lv), mode, st))
            _lib.check(lib.tdiff_set_fixed_tape(eng, _ptr(fix_pn), _ptr(fix_vu)))
        elif fixed_noise_tape is not None:
            raise ValueError('fixed_noise_tape without fixed_mask')
        if start_time is not None:
            st_pn = st_vu = None
            if start_noise_tape is not None:
                st_pn = start_noise_tape[0].detach().to(dev, torch.float32).contiguous()
                if tuple(st_pn.shape) != (Nl, 3):
                    raise ValueError('start noise tape positions must be [Nl,3] = %s, got %s' % ((Nl, 3), tuple(st_pn.shape)))
                if not pos_only:
                    st_vu = start_noise_tape[1].detach().to(dev, torch.float32).contiguous()
                    if tuple(st_vu.shape) != (Nl, K):
                        raise ValueError('start noise tape uniforms must be [Nl,K] = %s, got %s' % ((Nl, K), tuple(st_vu.shape)))
            _lib.check(lib.tdiff_set_start(eng, int(start_time), _ptr(st_pn), _ptr(st_vu)))
        if seed is None:        # with a tape the Philox key is unused: do not advance the caller's CPU generator (rng='cpu' driver parity)
            seed = 0 if noise_tape is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
        pos_traj = v_traj = v0_traj = vt_traj = None
        if return_traj:
            pos_traj = torch.empty(S, Nl, 3, device=dev)
            v_traj = torch.empty(S, Nl, dtype=torch.int64, device=dev)
            if not pos_only:
                v0_traj = torch.empty(S, Nl, K, device=dev)
                vt_traj = torch.empty(S, Nl, K, device=dev)
        if time_path is not None:
            _lib.check(lib.tdiff_sample_path(eng, _lib.i32_array(time_path), S, _ptr(pos_noise), _ptr(v_uniform), ctypes.c_uint64(seed),
                                             _ptr(pos_traj), _ptr(v_traj), _ptr(v0_traj), _ptr(vt_traj), int(bool(pos_only)), st))
        elif time_seq is None:
            _lib.check(lib.tdiff_sample(eng, S, _ptr(pos_noise), _ptr(v_uniform), ctypes.c_uint64(seed), _ptr(pos_traj), _ptr(v_traj),
                                        _ptr(v0_traj), _ptr(vt_traj), int(bool(pos_only)), st))
        else:
            _lib.check(lib.tdiff_sample_seq(eng, _lib.i32_array(time_seq), S, _ptr(pos_noise), _ptr(v_uniform), ctypes.c_uint64(seed),
                                            _ptr(pos_traj), _ptr(v_traj), _ptr(v0_traj), _ptr(vt_traj), int(bool(pos_only)), st))
        out_pos = torch.empty(Nl, 3, device=dev)
        out_v = torch.empty(Nl, dtype=torch.int64, device=dev)
        _lib.check(lib.tdiff_get_ligand(eng, _ptr(out_pos), _ptr(out_v), 1, st))
        if stack_traj:
            as_list = lambda t: t.cpu() if t is not None else None
        else:
            as_list = lambda t: list(t.cpu().unbind(0)) if t is not None else []  # one D2H per trajectory, not one per step
        return {'pos': out_pos, 'v': out_v, 'pos_traj': as_list(pos_traj), 'v_traj': as_list(v_traj), 'v0_traj': as_list(v0_traj),
                'vt_traj': as_list(vt_traj)}

    # ------------------------------------------------------------------ out of scope on this path
    def get_diffusion_loss(self, *a, **k):
        raise NotImplementedError('training is out of scope of the H100 sampling engine (SURVEY.md section 2)')

    # ------------------------------------------------------------------ second consumer of forward (SURVEY.md 8(f) n3)
    def _tab(self, name, t, batch):
        return getattr(self, name)[t][batch].unsqueeze(-1)

    def _q_v_pred(self, log_v0, t, batch, one_step=False):
        """log q(v_t | v_0) (or the single-step kernel), reference models/molopt_score_model.py:371-392"""
        la = self._tab('log_alphas_v' if one_step else 'log_alphas_cumprod_v', t, batch)
        l1 = self._tab('log_one_minus_alphas_v' if one_step else 'log_one_minus_alphas_cumprod_v', t, batch)
        x, y = log_v0 + la, l1 - math.log(self.num_classes)
        m = torch.max(x, y)
        return m + torch.log(torch.exp(x - m) + torch.exp(y - m))

    def _q_v_posterior(self, log_v0, log_vt, t, batch):
        un = self._q_v_pred(log_v0, (t - 1).clamp(min=0), batch) + self._q_v_pred(log_vt, t, batch, one_step=True)   # :401-409
        return un - torch.logsumexp(un, dim=-1, keepdim=True)

    def _log_onehot(self, idx):
        if int(idx.max()) >= self.num_classes:
            raise ValueError('atom-type index %d >= num_classes %d' % (int(idx.max()), self.num_classes))   # reference assert, :125
        return torch.log(F.one_hot(idx, self.num_classes).float().clamp(min=1e-30))

    @torch.no_grad()
    def likelihood_estimation(self, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step, noise=None):
        """Per-graph variational-bound terms (kl_pos, kl_v) at `time_step` [B], or the prior KL pair when `time_step == T`
        everywhere (reference models/molopt_score_model.py:565-617; caller scripts/likelihood_est_diffusion.py:30-40).
        The network evaluation is `forward` on libtdiff.so; the few [Nl,13]-sized formulas around it are torch elementwise ops
        on the caller's device.  `noise=(pos_noise [Nl,3], v_uniform [Nl,K])` replaces the two RNG draws (parity tests)."""
        from . import ops
        T, K = self.num_timesteps, self.num_classes
        dev = protein_pos.device
        time_step = time_step.to(dev, torch.long)
        B = int(batch_protein.max()) + 1
        if time_step.numel() != B:
            raise ValueError('time_step must have one entry per graph')
        offset = ops.scatter_mean3(protein_pos.float(), batch_protein)                      # center_pos(mode='protein'), :110-120
        protein_pos = protein_pos.float() - offset[batch_protein]
        x0 = ligand_pos.float() - offset[batch_ligand]
        cnt = torch.bincount(batch_ligand, minlength=B).clamp(min=1).float()
        graph_mean = lambda v: torch.zeros(B, device=dev).index_add_(0, batch_ligand, v) / cnt
        normal_kl = lambda m1, lv1, m2, lv2: (0.5 * (-1.0 + lv2 - lv1 + torch.exp(lv1 - lv2) + (m1 - m2) ** 2 * torch.exp(-lv2))).sum(-1)
        is_prior = bool((time_step == T).all())
        if not is_prior and not bool((time_step < T).all()):
            raise ValueError('time_step must be all == num_timesteps or all < num_timesteps')        # reference assert, :570
        if is_prior:
            last = torch.full((B,), T - 1, dtype=torch.long, device=dev)
            a_pos = self._tab('alphas_cumprod', last, batch_ligand)
            mean, logvar = a_pos.sqrt() * x0, torch.log((1.0 - a_pos).sqrt())
            kl_pos = graph_mean(normal_kl(torch.zeros_like(mean), torch.zeros_like(logvar), mean, logvar))
            log_qT = self._q_v_pred(self._log_onehot(batch_ligand), last, batch_ligand)          # graph ids as types, as the reference (:573)
            kl_v = graph_mean((log_qT.exp() * (log_qT + math.log(K))).sum(1))
            return kl_pos, kl_v
        if self.model_mean_type != 'C0':          # the reference raises here too (models/molopt_score_model.py:601-605); the prior branch above is mean-type free
            raise ValueError('likelihood_estimation needs model_mean_type C0, got %r' % (self.model_mean_type,))
        if noise is None:
            pos_noise = torch.randn_like(x0)
            v_uniform = torch.rand(x0.shape[0], K, device=dev)
        else:
            pos_noise, v_uniform = noise[0].to(dev, torch.float32), noise[1].to(dev, torch.float32)
        a_pos = self.alphas_cumprod.index_select(0, time_step)[batch_ligand].unsqueeze(-1)
        xt = a_pos.sqrt() * x0 + (1.0 - a_pos).sqrt() * pos_noise                                     # :583
        log_v0 = self._log_onehot(ligand_v)
        gumbel = -torch.log(-torch.log(v_uniform + 1e-30) + 1e-30)
        vt = (gumbel + self._q_v_pred(log_v0, time_step, batch_ligand)).argmax(dim=-1)                # q_v_sample, :394-398
        log_vt = self._log_onehot(vt)
        out = self.forward(protein_pos, protein_v, batch_protein, xt, vt, batch_ligand, time_step=time_step)
        c0 = self._tab('posterior_mean_c0_coef', time_step, batch_ligand)
        ct = self._tab('posterior_mean_ct_coef', time_step, batch_ligand)
        mean_model, mean_true = c0 * out['pred_ligand_pos'] + ct * xt, c0 * x0 + ct * xt              # q_pos_posterior, :424-428
        log_model = self._q_v_posterior(F.log_softmax(out['pred_ligand_v'], dim=-1), log_vt, time_step, batch_ligand)
        log_true = self._q_v_posterior(log_v0, log_vt, time_step, batch_ligand)
        decoder = (time_step == 0).float()[batch_ligand]
        logvar = self._tab('posterior_logvar', time_step, batch_ligand)
        kl_p = normal_kl(mean_true, logvar, mean_model, logvar) / math.log(2.)                        # compute_pos_Lt, :470-482
        ls = 0.5 * logvar
        nll_p = ((x0 - mean_model) ** 2 / (2 * torch.exp(2 * ls)) + ls + math.log(math.sqrt(2 * math.pi))).sum(-1)
        kl_pos = graph_mean(decoder * nll_p + (1. - decoder) * kl_p)
        kl_c = (log_true.exp() * (log_true - log_model)).sum(1)                                       # compute_v_Lt, :484-489
        nll_c = -(log_v0.exp() * log_model).sum(1)
        kl_v = graph_mean(decoder * nll_c + (1. - decoder) * kl_c)
        return kl_pos, kl_v

    @torch.no_grad()
    def likelihood_terms(self, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, time_step, keys=None, seed=None,
                         noise=None, return_atoms=False):
        """Variational-bound terms of every graph at its own `time_step` [B] (0..T-1) in one engine call (tdiff_likelihood_terms,
        DESIGN.md section 1): noising, the forward and the per-atom terms and per-graph means on the device, plus the prior terms of
        every graph with the ligand's own types.  The ligand is the clean one, in the lab frame; everything is centred on the protein.
        Noise comes from the engine's likelihood stream, keyed per graph by `keys` [B] (default: the graph index) and `seed` (default:
        drawn from torch's CPU generator), so a graph's terms do not depend on the rest of the batch; `noise=(pos_noise [Nl,3],
        v_uniform [Nl,K])` replaces it.  Returns device tensors kl_pos, kl_v, prior_pos, prior_v [B]; `return_atoms` adds atom_kl_pos,
        atom_kl_v [Nl], xt [Nl,3] (centred frame) and vt [Nl].  `likelihood_estimation` above stays the reference-signature entry with
        the reference's random stream and graph-id prior."""
        T, K = self.num_timesteps, self.num_classes
        if self.model_mean_type != 'C0':          # the reference raises (models/molopt_score_model.py:601-605)
            raise ValueError('likelihood_terms needs model_mean_type C0, got %r' % (self.model_mean_type,))
        ts = [int(x) for x in torch.as_tensor(time_step).reshape(-1).tolist()]
        if any(not 0 <= x <= T - 1 for x in ts):
            raise ValueError('time_step must lie in 0..T-1 = %d' % (T - 1))
        dev = protein_pos.device
        eng = self.engine(dev)
        lib = _lib.load()
        st = self._stream(dev)
        B, Np, Nl = self._bind(eng, protein_pos, protein_v, batch_protein, batch_ligand, 1)
        if len(ts) != B:
            raise ValueError('time_step must have one entry per graph: %d entries, %d graphs' % (len(ts), B))
        key_arr = None
        if keys is not None:
            kl = [int(x) for x in torch.as_tensor(keys).reshape(-1).tolist()]
            if len(kl) != B or any(not 0 <= x < 2 ** 32 for x in kl):
                raise ValueError('keys must be %d integers in 0..2^32-1' % B)
            key_arr = (ctypes.c_uint32 * B)(*kl)
        lpos = ligand_pos.detach().to(torch.float32).contiguous()
        lv = ligand_v.detach().to(torch.int64).contiguous()
        if lpos.shape[0] != Nl or lv.shape[0] != Nl:
            raise ValueError('ligand arrays disagree with batch_ligand')
        _lib.check(lib.tdiff_set_ligand(eng, _ptr(lpos), _ptr(lv), 1, st))
        pos_noise = v_uniform = None
        if noise is not None:
            pos_noise = noise[0].detach().to(dev, torch.float32).contiguous()
            v_uniform = noise[1].detach().to(dev, torch.float32).contiguous()
            if tuple(pos_noise.shape) != (Nl, 3) or tuple(v_uniform.shape) != (Nl, K):
                raise ValueError('noise shapes must be [Nl,3] = %s and [Nl,K] = %s, got %s and %s'
                                 % ((Nl, 3), (Nl, K), tuple(pos_noise.shape), tuple(v_uniform.shape)))
        if seed is None:        # as sample_diffusion: with a tape the key is unused and the caller's CPU generator is not advanced
            seed = 0 if noise is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
        out = {k: torch.empty(B, device=dev) for k in ('kl_pos', 'kl_v', 'prior_pos', 'prior_v')}
        atoms = {}
        if return_atoms:
            atoms = {'atom_kl_pos': torch.empty(Nl, device=dev), 'atom_kl_v': torch.empty(Nl, device=dev),
                     'xt': torch.empty(Nl, 3, device=dev), 'vt': torch.empty(Nl, dtype=torch.int64, device=dev)}
        _lib.check(lib.tdiff_likelihood_terms(eng, _lib.i32_array(ts), key_arr, _ptr(pos_noise), _ptr(v_uniform), ctypes.c_uint64(seed),
                                              _ptr(out['kl_pos']), _ptr(out['kl_v']), _ptr(out['prior_pos']), _ptr(out['prior_v']),
                                              _ptr(atoms.get('atom_kl_pos')), _ptr(atoms.get('atom_kl_v')), _ptr(atoms.get('xt')),
                                              _ptr(atoms.get('vt')), st))
        out.update(atoms)
        return out

    @torch.no_grad()
    def fetch_embedding(self, protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand):
        """reference models/molopt_score_model.py:619-631: forward with fix_x=True."""
        return self.forward(protein_pos, protein_v, batch_protein, ligand_pos, ligand_v, batch_ligand, fix_x=True)
