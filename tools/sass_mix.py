"""Developer tool (no GPU needed): the instruction mix the compiler made of a CUDA source's kernels.

Cross-compiles one source of nero_b200/csrc for sm_90a into a cubin with `-Xptxas -v`, then prints for each kernel
whose demangled name contains the filter: its ptxas register / spill lines and its SASS instruction counts by class
(integer ALU, IMAD, FP32, MUFU, global loads / stores, shared stores, ...).  Static counts of the code, not of what runs.

    python tools/sass_mix.py [--src k_gemm_chain.cu] [--filter gemm_chain_kernel] [--flags=-DNERO_CHAIN_PHASES] [--json]
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nero_b200 import build as B  # noqa: E402

CUDA_BIN = os.path.dirname(B.NVCC)
# opcode (without modifiers) -> class; anything else counts as 'other'
CLASSES = {
    'int': ('LOP3', 'LEA', 'IADD3', 'ISETP', 'PLOP3', 'SHF', 'FSEL', 'SEL', 'IABS', 'IMNMX', 'LOP', 'SGXT', 'BMSK', 'P2R', 'R2P'),
    'imad': ('IMAD',),
    'fp32': ('FADD', 'FMUL', 'FFMA', 'FMNMX', 'FSETP', 'FCHK', 'FRND'),
    'mufu': ('MUFU',),
    'cvt': ('F2F', 'F2FP', 'F2I', 'I2F', 'PRMT'),
    'ldg': ('LDG',),
    'stg': ('STG',),
    'sts': ('STS',),
    'lds': ('LDS', 'LDSM'),
    'local': ('LDL', 'STL'),
    'wgmma': ('HGMMA',),
    'branch': ('BRA', 'BSSY', 'BSYNC', 'WARPSYNC', 'EXIT', 'CALL', 'RET'),
    'move': ('MOV', 'S2R', 'S2UR', 'CS2R', 'R2UR', 'ULDC', 'UMOV', 'LDC'),
}
OPCLASS = {op: c for c, ops in CLASSES.items() for op in ops}
INSN = re.compile(r'/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[0-9T]+\s+)?([A-Z][A-Z0-9_]*)')


def compile_cubin(src, flags, out):
    cmd = [B.NVCC] + B.ARCH + ['-O3', '-std=c++17', '--expt-relaxed-constexpr', '-Xptxas', '-v', '-cubin'] + list(flags) + [
        '-o', out, os.path.join(B.CSRC, src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(r.stdout + r.stderr)
    return r.stdout + r.stderr


def demangle(names):
    r = subprocess.run([os.path.join(CUDA_BIN, 'cu++filt')], input='\n'.join(names), capture_output=True, text=True)
    return dict(zip(names, r.stdout.splitlines())) if r.returncode == 0 else {n: n for n in names}


def ptxas_lines(log):
    """mangled kernel name -> its ptxas resource lines (registers, spills)."""
    out, cur = collections.defaultdict(list), None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line) or re.search(r"Function properties for (\w+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and ('spill' in line or 'registers' in line):
            out[cur].append(line.split('ptxas info    :')[-1].strip())
    return out


def sass_mix(cubin):
    """mangled kernel name -> Counter of instruction classes (plus 'total')."""
    txt = subprocess.run([os.path.join(CUDA_BIN, 'cuobjdump'), '-sass', cubin], capture_output=True, text=True, check=True).stdout
    mix, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = mix.setdefault(m.group(1), collections.Counter())
            continue
        m = INSN.search(line)
        if cur is not None and m:
            op = m.group(1).split('.')[0]
            if op == 'NOP':
                continue
            cur['total'] += 1
            cur[OPCLASS.get(op, 'other')] += 1
    return mix


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--src', default='k_gemm_chain.cu')
    ap.add_argument('--filter', default='', help='keep kernels whose demangled name contains this')
    ap.add_argument('--flags', default='', help='extra nvcc flags, space separated')
    ap.add_argument('--json', action='store_true')
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, 'k.cubin')
        log = compile_cubin(a.src, a.flags.split(), cubin)
        mix = sass_mix(cubin)
    res = ptxas_lines(log)
    names = demangle(sorted(mix))
    cols = ['total', 'int', 'imad', 'fp32', 'mufu', 'cvt', 'ldg', 'stg', 'sts', 'local', 'wgmma', 'branch']
    rows = []
    for mangled in sorted(mix, key=lambda n: names[n]):
        if a.filter not in names[mangled]:
            continue
        rows.append({'kernel': names[mangled], 'ptxas': res.get(mangled, []), **{c: mix[mangled][c] for c in cols + ['other']}})
    if a.json:
        print(json.dumps(rows, indent=1))
        return
    for r in rows:
        print(r['kernel'])
        for line in r['ptxas']:
            print('   ', line)
        print('    ' + '  '.join(f'{c} {r[c]}' for c in cols + ['other']))


if __name__ == '__main__':
    main()
