"""CPU-side checks of the drop-in boundary: the shared library loads and exports every symbol include/tdiff.h declares,
the ctypes table covers exactly those, and without a GPU the engine fails loudly (no fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, 'include', 'tdiff.h')).read()
    return sorted(set(re.findall(r'^TDIFF_API [^;(]*?\b(tdiff_[a-z0-9_]+)\(', src, flags=re.M)))


def test_library_exports_every_declared_symbol():
    from targetdiff_b200 import _lib
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(_lib.SIGNATURES) == names
    assert b'sm_90a' in lib.tdiff_version()


@pytest.mark.skipif(torch.cuda.is_available(), reason='CPU-only behaviour')
def test_no_cpu_fallback():
    from targetdiff_b200 import _lib
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    lib = _lib.load()
    cfg = _lib.tdiff_config(128, 16, 9, 32, 20, 13, 27, 1000)
    out = ctypes.c_void_p()
    rc = lib.tdiff_create(ctypes.byref(cfg), (_lib.tdiff_tensor * 1)(), 0, 0, ctypes.byref(out))
    assert rc == _lib.TDIFF_ECUDA and b'no CPU fallback' in lib.tdiff_last_error()
    m = ScorePosNet3D(default_model_config(), 27, 13)
    z = torch.zeros
    with pytest.raises(RuntimeError, match='no CPU path'):
        m(z(3, 3), z(3, 27), z(3, dtype=torch.long), z(1, 3), z(1, dtype=torch.long), z(1, dtype=torch.long))
    with pytest.raises(RuntimeError, match='no CPU path'):
        m.sample_diffusion(z(3, 3), z(3, 27), z(3, dtype=torch.long), z(1, 3), z(1, dtype=torch.long), z(1, dtype=torch.long), num_steps=2)


def test_state_dict_layout_and_unsupported_configs():
    from oracle import restate, synth
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    m = ScorePosNet3D(default_model_config(), 27, 13)
    sd = m.state_dict()
    spec = synth.state_dict_spec()
    assert list(sd.keys()) == [k for k, _, _ in spec]
    assert all(tuple(sd[k].shape) == tuple(s) for k, s, _ in spec)
    sched = restate.make_schedules()
    assert all(torch.equal(sd[k], sched[k]) for k in synth.SCHEDULE_KEYS)
    m.load_state_dict(synth.make_state_dict(0, schedules=sched), strict=True)
    for bad in ({'cutoff_mode': 'radius'}, {'model_type': 'egnn'}, {'time_emb_dim': 8, 'time_emb_mode': 'sin'},
                {'num_blocks': 0}, {'hidden_dim': 256}, {'ew_net_type': 'x'}):
        c = default_model_config()
        c.update(bad)
        with pytest.raises(NotImplementedError):
            ScorePosNet3D(c, 27, 13)
    # the backbone options of SURVEY 8(f) n2 are accepted and give the reference's state_dict layout (key order and shapes)
    for opt in ({'num_blocks': 2}, {'ew_net_type': 'r'}, {'ew_net_type': 'm'}, {'ew_net_type': 'none'}, {'x2h_out_fc': True},
                {'time_emb_dim': 1, 'time_emb_mode': 'simple'}, {'cutoff_mode': 'hybrid'}):
        c = default_model_config()
        c.update(opt)
        m = ScorePosNet3D(c, 27, 13)
        spec = synth.state_dict_spec(opt)
        assert list(m.state_dict().keys()) == [k for k, _, _ in spec], opt
        assert all(tuple(m.state_dict()[k].shape) == tuple(s) for k, s, _ in spec), opt


def test_config_struct_matches_header():
    """The ctypes mirror of `tdiff_config` has the header's fields in the header's order and the same size (16 x int32)."""
    from targetdiff_b200 import _lib
    src = open(os.path.join(ROOT, 'include', 'tdiff.h')).read()
    body = src[src.index('typedef struct tdiff_config {'):src.index('} tdiff_config;')]
    fields = re.findall(r'^\s*int32_t\s+([a-z0-9_]+)(\[(\d+)\])?;', body, flags=re.M)
    names = [f[0] for f in fields]
    words = sum(int(f[2]) if f[2] else 1 for f in fields)
    assert names == [n for n, _ in _lib.tdiff_config._fields_]
    assert ctypes.sizeof(_lib.tdiff_config) == 4 * words == 64
    assert names.index('model_mean_type') == 8 and names[-1] == 'reserved'


def test_model_mean_type_reaches_the_engine_config():
    from targetdiff_b200.config import default_model_config
    from targetdiff_b200.score_model import ScorePosNet3D
    for name in ('C0', 'noise'):
        c = default_model_config()
        c.update({'model_mean_type': name})
        assert ScorePosNet3D(c, 27, 13).model_mean_type == name
    c = default_model_config()
    c.update({'model_mean_type': 'x0'})
    with pytest.raises(NotImplementedError):
        ScorePosNet3D(c, 27, 13)
