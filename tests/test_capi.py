"""The C-ABI library loads and exports every symbol include/serl_b200.h declares (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_text():
    """include/serl_b200.h without its comments"""
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'serl_b200.h')).read(), flags=re.S)


def declared_symbols():
    return sorted(set(re.findall(r'\b(serl_[a-z0-9_]+)\s*\(', header_text())))


def declared_prototypes():
    """{entry point: (result type, [parameter declarations])} of every prototype in the header"""
    protos = {}
    for ret, name, params in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', header_text()):
        params = [p.strip() for p in params.split(',')]
        protos[name] = (ret.strip(), [] if params == ['void'] else params)
    return protos


_SCALARS = {'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64, 'double': ctypes.c_double, 'float': ctypes.c_float,
            'int': ctypes.c_int}


def _matches(decl, ctype, is_param):
    """does ctypes type `ctype` have the C kind of the declaration `decl` (a parameter with its name, or a result type)?"""
    decl = re.sub(r'\s*\*', '*', decl)
    if decl.startswith('const char*'):
        return ctype is ctypes.c_char_p
    if decl.startswith('void*'):
        return ctype is ctypes.c_void_p
    if '*' in decl:
        return ctype is ctypes.c_void_p or issubclass(ctype, ctypes._Pointer)
    if decl == 'void':
        return ctype is None
    return ctype is _SCALARS[decl.split()[-2] if is_param else decl]


def test_binding_declares_every_entry_point_with_the_header_signature():
    """_native.SIGNATURES (read without loading the library) against every prototype of include/serl_b200.h: the same entry
    points, the same number of arguments and the same C kind for each argument and for the result."""
    from serl_b200 import _native
    protos = declared_prototypes()
    assert len(protos) == len(declared_symbols()) == 21
    assert sorted(_native.SIGNATURES) == sorted(protos)
    for name, (ret, params) in protos.items():
        restype, argtypes = _native.SIGNATURES[name]
        assert _matches(ret, restype, False), (name, ret, restype)
        assert len(argtypes) == len(params), (name, params, argtypes)
        for decl, t in zip(params, argtypes):
            assert _matches(decl, t, True), (name, decl, t)


def test_library_exports_all_declared_symbols():
    from serl_b200 import build, _native
    build.build()
    lib = ctypes.CDLL(_native.LIB_PATH)
    syms = declared_symbols()
    assert 'serl_rollout' in syms
    for s in syms:
        assert hasattr(lib, s), s


def test_num_params_matches_reference_formula():
    from serl_b200 import rollout
    for h, p in ((32, 3715), (72, 16995), (96, 29571), (128, 51715)):   # SURVEY 8(a): P = 3h^2 + 20h + 3
        assert rollout.num_params(rollout.actor_shape(h)) == p


def test_compute_fails_loudly_without_cuda():
    import torch
    from serl_b200 import rollout, _native
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    sh = rollout.actor_shape(32)
    w = torch.zeros((1, rollout.num_params(sh)))
    with pytest.raises(_native.NativeError):
        rollout.population_rollout(w, sh, torch.zeros((1, 2, 6), dtype=torch.float64), torch.zeros((1, 2, 6), dtype=torch.float64),
                                   torch.zeros(1, dtype=torch.int32))


@pytest.mark.parametrize('widths', [None, [128, 128]])
def test_rollout_run_rejects_a_bad_descriptor_before_any_cuda_call(widths):
    """Both kernels (K1 and, with widths, K1-TC) go through the same checks; the device pointers are never dereferenced."""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    warr = (ctypes.c_int32 * 2)(*(widths or [0, 0]))

    def run(**kw):
        d = _native.RolloutDesc()
        fake = iter(range(0x10000, 0x100000, 0x1000))      # non-null, never read
        for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_fitness', 'd_replay', 'd_status'):
            setattr(d, f, next(fake))
        d.pop, d.shape, d.n_envs, d.horizon, d.replay_env = 4, rollout.actor_shape(72), 8, 100, 0
        if widths:
            d.widths, d.n_widths = ctypes.cast(warr, ctypes.c_void_p), 2
        for k, v in kw.items():
            setattr(d, k, v)
        return L.serl_rollout_run(ctypes.byref(d), None), L.serl_last_error().decode()

    rc, msg = run(replay_env=8)
    assert rc == -1 and 'replay_env' in msg, (rc, msg)
    assert run(pop=0)[0] == -1
    assert run(shape=_native.ActorShape(7, 3, 72, 3, 5))[0] == -1          # activation 5


def test_ctypes_mirror_of_the_rollout_descriptor_matches_the_header(tmp_path):
    """serl_b200/_native.py RolloutDesc / ActorShape vs include/serl_b200.h: same size and same field offsets (gcc); every header
    constant _native restates (enum orders, record widths, env_mode and flag bits) and the env_mode decoders of rollout.py."""
    import subprocess
    from serl_b200 import _native, rollout
    fields = [f for f, _ in _native.RolloutDesc._fields_]
    names = sorted(set(re.findall(r'\b(SERL_(?:PLANT|FAULT|ACT|STATUS)_[A-Z0-9_]+)\s*=', header_text())))
    names += ['SERL_TRACE_COLS', 'SERL_REPLAY_COLS', 'SERL_MODE_GUST', 'SERL_MODE_GUST_UP', 'SERL_ROLLOUT_GUST']
    src = tmp_path / 'layout.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "serl_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu\\n", sizeof(serl_rollout_desc), sizeof(serl_actor_shape));\n' +
                   ''.join('  printf("%%zu\\n", offsetof(serl_rollout_desc, %s));\n' % f for f in fields) +
                   ''.join('  printf("%s %%lld\\n", (long long)%s);\n' % (n, n) for n in names) + '  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).splitlines()
    size, shape_size = map(int, out[0].split())
    assert size == ctypes.sizeof(_native.RolloutDesc) and shape_size == ctypes.sizeof(_native.ActorShape)
    for f, line in zip(fields, out[1:]):
        assert int(line) == getattr(_native.RolloutDesc, f).offset, f
    c = {k: int(v) for k, v in (line.split() for line in out[1 + len(fields):])}
    assert len(c) == len(names)
    plants = {k[len('SERL_PLANT_'):].lower(): v for k, v in c.items() if k.startswith('SERL_PLANT_') and k != 'SERL_PLANT_COUNT'}
    assert plants == {v: i for i, v in enumerate(_native.PLANT_VARIANTS)} and c['SERL_PLANT_COUNT'] == len(_native.PLANT_VARIANTS)
    assert {k[len('SERL_FAULT_'):].lower(): v for k, v in c.items() if k.startswith('SERL_FAULT_')} == \
        {f: i for i, f in enumerate(_native.FAULTS)}
    assert {k: v for k, v in c.items() if k.startswith('SERL_ACT_')} == \
        {'SERL_ACT_TANH': _native.ACTIVATIONS['tanh'], 'SERL_ACT_ELU': _native.ACTIVATIONS['elu'],
         'SERL_ACT_LEAKY_RELU': _native.ACTIVATIONS['relu']}
    assert len(_native.ACTIVATIONS) == 3
    assert (c['SERL_TRACE_COLS'], c['SERL_REPLAY_COLS']) == (_native.TRACE_COLS, _native.REPLAY_COLS)
    assert (c['SERL_MODE_GUST'], c['SERL_MODE_GUST_UP'], c['SERL_ROLLOUT_GUST']) == (rollout.MODE_GUST, rollout.MODE_GUST_UP, _native.ROLLOUT_GUST)
    assert {k: v for k, v in c.items() if k.startswith('SERL_STATUS_')} == \
        {'SERL_STATUS_NONFINITE': _native.STATUS_NONFINITE, 'SERL_STATUS_GUST_FLAG': _native.STATUS_GUST_FLAG}
    assert rollout.REPLAY_COST == rollout.TRANSITION_COLS == _native.REPLAY_COLS - 1
    assert rollout.mode_code('gust') == rollout.mode_code('nominal') | rollout.MODE_GUST
    assert rollout.mode_code('cg-timed') >> 16 == rollout.PLANT_VARIANTS.index('cg_timed_post')
    code = c['SERL_PLANT_CG_TIMED'] | c['SERL_FAULT_SE'] << 8 | c['SERL_PLANT_CG_TIMED_POST'] << 16 | c['SERL_MODE_GUST']
    assert rollout.mode_variant(code) == c['SERL_PLANT_CG_TIMED'] and rollout.mode_gust(code)
    assert rollout.timed_plant_code(code) == code - (c['SERL_FAULT_SE'] << 8)
    assert rollout.timed_plant_code(c['SERL_PLANT_ICE'] | c['SERL_FAULT_BE'] << 8) is None
