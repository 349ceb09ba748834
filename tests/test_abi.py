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


def test_header_structs_match_the_library():
    """The structs the bindings read from the header have the sizes the library was compiled with, and the numpy job
    records have the sizes of their structs."""
    from nero_b200 import ops
    lib = ops.lib
    assert len(ops.ABI_RECORDS) == 7
    for i, name in enumerate(ops.ABI_RECORDS):
        assert lib.nero_abi_sizeof(i) == ctypes.sizeof(ops.STRUCTS[name]), name
    assert lib.nero_abi_sizeof(len(ops.ABI_RECORDS)) == -1 and lib.nero_abi_sizeof(99) == -1
    assert ops._PREP_JOB.itemsize == lib.nero_abi_sizeof(4) and ops._FINISH_JOB.itemsize == lib.nero_abi_sizeof(3)


def test_every_entry_point_has_its_header_prototype():
    """Each prototype of the header is set on the library with one argtype per parameter; a call that does not match it is
    refused before it reaches C."""
    import pytest
    from nero_b200 import ops
    txt = re.sub(r'/\*.*?\*/', ' ', open(os.path.join(ROOT, 'include', 'nero_b200.h')).read(), flags=re.S)
    protos = dict(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(([^)]*)\)', txt))
    assert len(protos) == len(declared_symbols()) == 57
    for name, params in protos.items():
        n = 0 if params.strip() in ('', 'void') else params.count(',') + 1
        fn = getattr(ops.lib, name)
        assert fn.argtypes is not None and len(fn.argtypes) == n and fn.restype is ctypes.c_int, name
    assert ops.lib.nero_abi_sizeof(2) > 0
    with pytest.raises(ctypes.ArgumentError):
        ops.lib.nero_abi_sizeof(2.0)
