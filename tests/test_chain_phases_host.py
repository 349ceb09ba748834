"""CPU: the fused chain's phase-timer pointer is part of the C ABI, and the product library's chain kernels carry no timer
code (only the NERO_CHAIN_PHASES diagnostic build of tools/chain_phases.py reads the clocks)."""
import ctypes
import re
import subprocess


def test_chain_params_end_with_the_phase_counter_pointer():
    from nero_b200 import ops
    P = ops.ChainParams
    names = [f[0] for f in P._fields_]
    assert names[-1] == 'phase_clk' and P._fields_[-1][1] is ctypes.c_void_p
    assert P.phase_clk.offset == ctypes.sizeof(P) - ctypes.sizeof(ctypes.c_void_p)
    assert ops.lib.nero_abi_sizeof(ops.ABI_RECORDS.index('nero_chain_params')) == ctypes.sizeof(P)
    assert ops.CHAIN_PHASES is None and P().phase_clk is None


def test_product_chain_kernels_have_no_timer_reads():
    import __graft_entry__ as g
    sass = subprocess.run(['cuobjdump', '-sass', g.build()], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r'\n\s*Function : ', sass)
    chain = [f for f in funcs if f.startswith('_ZN4nero17gemm_chain_kernel')]
    assert len(chain) == 3
    for f in chain:
        assert 'SR_CLOCK' not in f and 'SR_GLOBALTIMER' not in f, f.split('\n', 1)[0]
