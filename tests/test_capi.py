"""The C-ABI library loads and exports every symbol include/serl_b200.h declares (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, 'include', 'serl_b200.h')).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    return sorted(set(re.findall(r'\b(serl_[a-z0-9_]+)\s*\(', txt)))


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
    """serl_b200/_native.py RolloutDesc / ActorShape vs include/serl_b200.h: same size and same field offsets (gcc)."""
    import subprocess
    from serl_b200 import _native
    fields = [f for f, _ in _native.RolloutDesc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "serl_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu\\n", sizeof(serl_rollout_desc), sizeof(serl_actor_shape));\n' +
                   ''.join('  printf("%%zu\\n", offsetof(serl_rollout_desc, %s));\n' % f for f in fields) +
                   '  printf("%d %d %d %d\\n", SERL_ROLLOUT_GUST, SERL_MODE_GUST, SERL_STATUS_NONFINITE, SERL_STATUS_GUST_FLAG);\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).split('\n')
    size, shape_size = map(int, out[0].split())
    assert size == ctypes.sizeof(_native.RolloutDesc) and shape_size == ctypes.sizeof(_native.ActorShape)
    for f, line in zip(fields, out[1:]):
        assert int(line) == getattr(_native.RolloutDesc, f).offset, f
    from serl_b200 import rollout
    assert list(map(int, out[1 + len(fields)].split())) == [_native.ROLLOUT_GUST, rollout.MODE_GUST, _native.STATUS_NONFINITE, _native.STATUS_GUST_FLAG]
    assert rollout.mode_code('gust') == rollout.mode_code('nominal') | rollout.MODE_GUST
    assert rollout.mode_code('cg-timed') >> 16 == rollout.PLANT_VARIANTS.index('cg_timed_post')
