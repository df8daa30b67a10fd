"""The C-ABI shared library loads without a GPU and exports every symbol include/diffsampler_b200.h declares;
the ctypes struct mirrors have the compiled sizes.  No compute calls here."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def built():
    import __graft_entry__ as g
    mod = g._load_build_module()
    return mod.build()


def declared_symbols():
    src = open(os.path.join(ROOT, 'include', 'diffsampler_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(ds_[a-z0-9_]+)\s*\(', src)))


def test_header_symbols_exported(built):
    lib = ctypes.CDLL(built)
    names = declared_symbols()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f'{n} declared in the header but not exported'


def test_binding_lists_every_declared_symbol(built):
    from diff_sampler_b200 import _lib
    assert set(declared_symbols()) == set(_lib.EXPORTS)


def test_struct_mirrors_and_version(built):
    from diff_sampler_b200 import _lib
    assert 'sm_90a' in _lib.version()          # load() verifies every sizeof


def test_no_cpu_fallback(built):
    import torch
    from diff_sampler_b200 import solvers, solver_utils
    from diff_sampler_b200._lib import DsError
    with pytest.raises(RuntimeError):
        solvers.euler_sampler(lambda x, t, **k: x, torch.randn(2, 3, 8, 8), num_steps=3)
    with pytest.raises(DsError):
        solver_utils.solver_update(torch.zeros(2, 4), torch.zeros(2, 4), [1.0])


def test_oracle_is_not_imported_by_the_product():
    import subprocess
    import sys
    code = ("import sys; sys.path.insert(0, %r); import diff_sampler_b200.solvers, diff_sampler_b200.solvers_amed, "
            "diff_sampler_b200.gits_utils, diff_sampler_b200.net, diff_sampler_b200.plan; "
            "assert not [m for m in sys.modules if m.split('.')[0] == 'oracle'], 'product imports oracle'") % ROOT
    subprocess.run([sys.executable, '-c', code], check=True)
