"""Instruction footprint of one sparse-kernel iteration (CPU only: nvcc + nvdisasm, no GPU).

    python tools/sass_footprint.py [csrc_dir]

Compiles omg_b200.cu to an sm_90a cubin with the Makefile's flags and attributes the SASS of
omg_ipm_kernel_sp to source lines (nvdisasm -gi: the outermost line of every inlined call).
The per-iteration range runs from the first instruction of pass I1 to the last instruction of
the accept pass I12; every iteration walks through it once.  Bytes are split by the phases of
the TICK counters in ipm_body_sp (the same phases tools/sp_phases.py times).  Out-of-line
functions called from the range are listed with their sizes: they are walked as well, but only
one copy of each."""
import collections
import os
import re
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), 'omg_tools_b200', 'csrc')
CUDA = os.environ.get('CUDA_HOME', '/usr/local/cuda')
NVCC = os.environ.get('NVCC') or shutil.which('nvcc') or os.path.join(CUDA, 'bin', 'nvcc')
NVDISASM = os.path.join(os.path.dirname(NVCC), 'nvdisasm')
KERNEL = '_Z17omg_ipm_kernel_sp6DevTab5SpTab11omg_options5Batch6SpSmem'
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xptxas', '-v']
# phase k ends at TICK(k) (ipm_body_sp); the accept pass ends with the iteration loop
PHASES = {1: 'I1', 2: 'I2', 3: 'I3', 4: 'I4', 5: 'H gather', 6: 'W+border+rhs+staging', 7: 'factorisation',
          10: 'backward sweep', 11: 'I10', 12: 'I11 line search', 0: 'I12 accept'}


def compile_cubin(csrc, out_dir):
    """cubin path and the ptxas report (registers, stack, spills per function)."""
    cubin = os.path.join(out_dir, 'omg_b200.cubin')
    p = subprocess.run([NVCC] + FLAGS + ['-cubin', '-o', cubin, os.path.join(csrc, 'omg_b200.cu')],
                       cwd=csrc, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(p.stderr)
    return cubin, ptxas_report(p.stderr)


def ptxas_report(text):
    rep, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '?([\w$.]+)'?", line)
        if m:
            cur = rep.setdefault(m.group(1), {})
            continue
        if cur is None:
            continue
        m = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m:
            cur.update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
        m = re.search(r'Used (\d+) registers', line)
        if m:
            cur['regs'] = int(m.group(1))
    return rep


def sections(cubin):
    """{section: [(address, opcode text, [(file, line), ...] innermost to outermost)]}; a
    subroutine label inside a section is an entry (None, label, None)"""
    txt = subprocess.run([NVDISASM, '-gi', cubin], capture_output=True, text=True, check=True).stdout
    out, cur, chain, fresh = {}, None, [], True
    for line in txt.splitlines():
        m = re.match(r'//-+ \.text\.(\S+) -+', line)
        if m:
            cur = out.setdefault(m.group(1), [])
            chain = []
            continue
        m = re.match(r'(\$\S+):$', line)
        if m and cur is not None:        # a subroutine: the name holds until the next one
            cur.append((None, m.group(1), None))
            continue
        if line.startswith('//-'):
            cur = None
            continue
        if cur is None:
            continue
        if line.lstrip().startswith('//## File'):
            # one line per inlining level: "line a inlined at ... line b", then "line b inlined at ..."
            if fresh:
                chain, fresh = [], False
            chain += [(os.path.basename(f), int(n)) for f, n in re.findall(r'File "([^"]*)", line (\d+)', line)]
            chain += [(os.path.basename(f), int(n)) for f, n in re.findall(r'inlined at "([^"]*)", line (\d+)', line)]
            continue
        m = re.match(r'\s+/\*([0-9a-f]{4,})\*/\s+(.*)', line)
        if m:
            cur.append((int(m.group(1), 16), m.group(2), chain))
            fresh = True
    return out


def phase_lines(src):
    """line ranges of the iteration phases in omg_sp.cuh: {k: (first, last)} and the range"""
    lines = src.splitlines()
    body = next(i for i, l in enumerate(lines) if 'void ipm_body_sp(' in l)
    ticks = {}
    for i in range(body, len(lines)):
        m = re.search(r'\bTICK\((\d+)\)', lines[i])
        if m and int(m.group(1)) not in ticks:
            ticks[int(m.group(1))] = i + 1
        if '}  // iterations' in lines[i]:
            end = i + 1
            break
    order = sorted((ln, k) for k, ln in ticks.items() if k in PHASES and k != 0)
    rng, prev = {}, ticks[0]
    for ln, k in order:
        rng[k] = (prev + 1, ln)
        prev = ln
    rng[0] = (prev + 1, end)
    return rng, (ticks[0] + 1, end)


def footprint(csrc=CSRC):
    with open(os.path.join(csrc, 'omg_sp.cuh')) as f:
        prng, (lo, hi) = phase_lines(f.read())
    with tempfile.TemporaryDirectory() as d:
        cubin, rep = compile_cubin(csrc, d)
        secs = sections(cubin)
    # subroutines of the kernel's section (out-of-line functions, math-library slow paths)
    sub, name = collections.Counter(), None
    ins = []
    for e in secs[KERNEL]:
        if e[0] is None:
            name = e[1]
            continue
        ins.append(e + (name,))
        if name:
            sub[name] += 16

    def line(chain):                     # outermost line of ipm_body_sp's iteration loop
        for f, ln in reversed(chain or []):
            if f == 'omg_sp.cuh' and lo <= ln <= hi:
                return ln
        return None
    inside = [k for k, e in enumerate(ins) if e[3] is None and line(e[2])]
    rng = ins[inside[0]:inside[-1] + 1]
    per = collections.Counter()
    for _, op, chain, _ in rng:
        ln = line(chain)
        per[next((PHASES[k] for k, (p, q) in prng.items() if ln and p <= ln <= q), 'other')] += 16
    calls = collections.Counter(m for _, op, _, _ in rng for m in re.findall(r'CALL\.\S+ `\((\S+?)\)', op))
    callees = sorted(calls)
    return {
        'kernel_bytes': 16 * len(ins),
        'range_bytes': 16 * len(rng),
        'range_start': rng[0][0], 'range_end': rng[-1][0] + 16,
        'phases': per,
        'stl': sum(1 for e in rng if re.match(r'(@\S+\s+)?STL\b', e[1])),
        'ldl': sum(1 for e in rng if re.match(r'(@\S+\s+)?LDL\b', e[1])),
        'callees': {c: sub.get(c, 0) for c in callees},
        'calls': calls,                  # call sites in the range per out-of-line function
        'ptxas': rep.get(KERNEL, {}),
        'others': {k: 16 * sum(1 for e in v if e[0] is not None)
                   for k, v in secs.items() if 'omg_ipm_kernel' in k and k != KERNEL},
    }


def main():
    r = footprint(sys.argv[1] if len(sys.argv) > 1 else CSRC)
    p = r['ptxas']
    print('omg_ipm_kernel_sp: %d bytes of SASS; %s registers, %s bytes stack, spill stores %s / loads %s bytes'
          % (r['kernel_bytes'], p.get('regs'), p.get('stack'), p.get('spill_st'), p.get('spill_ld')))
    print('per-iteration range: %d bytes (0x%x..0x%x), STL %d, LDL %d'
          % (r['range_bytes'], r['range_start'], r['range_end'], r['stl'], r['ldl']))
    for name in list(PHASES.values()) + ['other']:
        print('  %-22s %8d' % (name, r['phases'].get(name, 0)))
    print('out-of-line functions called from the range (bytes, call sites):')
    for c, s in r['callees'].items():
        print('  %-60s %8d %4d' % (c.split('$')[-1], s, r['calls'][c]))
    print('other kernels (bytes of SASS):')
    for k, s in sorted(r['others'].items()):
        print('  %-60s %8d' % (k, s))


if __name__ == '__main__':
    main()
