"""CPU: the C-ABI library builds, loads, and exports every symbol include/nero_b200.h declares; the product package
refuses to run without it (no fallback).  No compute calls (no GPU here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, 'include', 'nero_b200.h')).read()
    return sorted(set(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(', txt)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    lib_path = g.build()
    lib = ctypes.CDLL(lib_path)
    syms = declared_symbols()
    assert len(syms) >= 28
    for s in syms:
        assert hasattr(lib, s), f'{s} declared in include/nero_b200.h but not exported'
    assert lib.nero_version() >= 100


def test_no_cpu_fallback():
    import pytest
    import torch
    from nero_b200.renderer import NeROShapeRenderer
    net = NeROShapeRenderer({'n_samples': 16, 'n_importance': 16}, training=False)
    o = torch.zeros(4, 3)
    with pytest.raises(RuntimeError):
        net.sample_ray(o, o, o[:, :1], o[:, :1], 0)


def test_sass_uses_hopper_tensor_path():
    """cuobjdump: the library is sm_90a code and contains HGMMA (wgmma.mma_async) and UBLKCP (bulk copy)."""
    import subprocess
    import __graft_entry__ as g
    lib = g.build()
    out = subprocess.run(['cuobjdump', '-sass', lib], capture_output=True, text=True).stdout
    for mnemonic in ('HGMMA', 'UBLKCP'):
        assert mnemonic in out, mnemonic
    assert 'HMMA.' not in out.replace('HGMMA', ''), 'legacy mma.sync path must not be used'
    elfs = subprocess.run(['cuobjdump', '-lelf', lib], capture_output=True, text=True).stdout.split()
    cubins = [e for e in elfs if e.endswith('.cubin')]
    assert cubins and all(e.endswith('.sm_90a.cubin') for e in cubins), cubins


def test_binding_struct_layouts_match_the_library():
    """ctypes / numpy mirrors of the structures that cross the C ABI have the sizes the library was compiled with."""
    import numpy as np
    from nero_b200 import ops
    lib = ops.lib
    assert lib.nero_abi_sizeof(0) == ctypes.sizeof(ops._ChainLayer)
    assert lib.nero_abi_sizeof(1) == ctypes.sizeof(ops._ChainParams)
    assert lib.nero_abi_sizeof(2) == ctypes.sizeof(ops.McParams)
    assert lib.nero_abi_sizeof(3) == ops._finish_job_dtype().itemsize
    assert lib.nero_abi_sizeof(4) == 88 and lib.nero_abi_sizeof(99) == -1
