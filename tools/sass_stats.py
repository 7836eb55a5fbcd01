#!/usr/bin/env python
"""Static per-phase / per-pipe instruction counts of the fused bootstrap kernel, from the SASS of the built
library (no GPU needed).  The NTT step is bound by the integer ALU pipe, so the ALU column of its step loop is
the number that predicts its run time; use this to judge an arithmetic change before spending GPU minutes.
The default kernel is the one the benchmark's workload launches: the throughput shape with the FP64 step
(`br_fft_step`, BrFft); its FP64 instructions (DADD / DMUL / DFMA, 2 cycles per warp-instruction on an H100 SXM SM
sub-partition) are counted in the `fp64` column.  The NTT throughput shape is
`--kernel blind_rotate_kernelINS_5BrCfgILi2ELi256ELi2ELb0ELb0EEELb0E`.  Every shape has a gate instantiation (`...Lb0E`
after the shape) and a lookup-table one (`...Lb1E`, kernels.cuh: LUT); give enough of the name to select one.

    python tools/sass_stats.py [--kernel blind_rotate_kernel] [--by-func] [--lib path/to/lib.so]

Each SASS instruction is attributed (through nvdisasm's inline chains, the library is built with -lineinfo)
to the line of `br2_step` (or `br_fft_step`) in kernels.cuh that called it, i.e. to a phase.  Counts are static: fwd1 / fwd2 /
fwd3 of the NTT step are multiplied by their two sweeps per step (the `it` loops are not unrolled), the MAC by its
two row iterations, and code inside the warp-uniform `switch (g)` of fwd2 / inv2 counts a quarter; the FP64 step
runs each of its five phases once per thread, with a real loop of four iterations inside pass 3
-- see `per step`.
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ALU = ('IADD3', 'IADD', 'LOP3', 'SHF', 'SEL', 'ISETP', 'PRMT', 'VIADD', 'LEA', 'IMNMX', 'VIMNMX', 'MOV', 'PLOP3', 'P2R',
       'R2P', 'IABS', 'FLO', 'POPC', 'BREV', 'SGXT', 'BMSK', 'LOP', 'FSEL', 'FMNMX', 'CS2R', 'VABSDIFF', 'FSETP', 'I2FP')
FMA = ('IMAD', 'FFMA', 'FMUL', 'FADD', 'HFMA2', 'IDP')
LSU = ('LDS', 'STS', 'LDG', 'STG', 'LD', 'ST', 'LDSM', 'ATOMS', 'ATOMG', 'RED', 'LDC', 'LDCU', 'UBLKCP', 'SYNCS')
FP64 = ('DADD', 'DMUL', 'DFMA', 'DSETP', 'DMNMX', 'F2F', 'F2I', 'I2F')
UNI = ('UMOV', 'UIADD3', 'ULEA', 'ULOP3', 'UISETP', 'USHF', 'UIMAD', 'S2UR', 'UPLOP3', 'USEL', 'UPRMT', 'R2UR', 'UFLO',
       'UP2UR', 'UIADD')


def pipe_of(op):
    base = op.split('.')[0]
    if base in ALU:
        return 'alu'
    if base in FMA:
        return 'fma'
    if base in LSU:
        return 'lsu'
    if base in UNI:
        return 'uni'
    if base in FP64:
        return 'fp64'
    return 'other'


COST = {'IMAD.WIDE(+R64)': 4, 'IMAD.WIDE(+RZ)': 4}
STEP_MULT = {'phase_fwd1': 2, 'phase_fwd2': 2, 'phase_fwd3': 2, 'phase_mac': 2,
             # the FP64 step (2 ciphertexts on 256 threads): one task per thread in each of its five phases; pass 3's
             # output-spectrum loop (fft_phase_mac) is weighted by `four_lines`
             'fft_phase_fwd1': 1, 'fft_phase_fwd2': 1, 'fft_phase_mac': 1, 'fft_phase_inv2': 1, 'fft_phase_inv1': 1}


def instruction_form(op, rest):
    """Opcode with the distinctions that matter for issue cost: carry-out predicates, 64-bit addends."""
    carry_out = bool(re.match(r'\s*R\w+, P\d', rest))
    if op.startswith('IMAD.WIDE'):
        key = 'IMAD.WIDE(+RZ)' if rest.rstrip(' ;').endswith('RZ') else 'IMAD.WIDE(+R64)'
    elif op.startswith('IADD3'):
        key = 'IADD3.X' if '.X' in op else 'IADD3'
    elif op.startswith('IMAD.HI'):
        key = 'IMAD.HI'
    else:
        key = re.sub(r'\.(LUT|U32|AND|OR|EX|GE|GT|LT|LE|NE|EQ|W|L|R|HI|64|128|E|CONSTANT|RECONVERGENT)\b', '', op)
    return key + ('.P' if carry_out and key.startswith(('IMAD', 'IADD3')) else '')


def enclosing_functions(path):
    """line -> name of the enclosing function (rough: last line that looks like a definition at depth <= 1)."""
    names = {}
    cur = None
    rx = re.compile(r'^\s*(?:template\s*<[^>]*>\s*)?(?:NB_HD|NB_D|NB_HDC|__global__|__device__)\b.*?\b([A-Za-z_][A-Za-z0-9_]*)\s*\(')
    try:
        with open(path) as f:
            for i, line in enumerate(f, 1):
                m = rx.match(line)
                if m:
                    cur = m.group(1)
                names[i] = cur
    except OSError:
        pass
    return names


def step_loop(kernel_ins, loop_addrs, labels):
    """The rotating step loop: from the target of its back-edge (the first backward branch after the last instruction of
    a step phase) to that branch.  Returns its size and the static count of spill (LDL / STL) and FP64 conversion
    (I2F.F64 / F2I.*F64) instructions inside it, or None if there is no such loop."""
    if not loop_addrs:
        return None
    last = max(loop_addrs)
    for addr, op, rest in kernel_ins:
        if addr < last or not op.startswith('BRA'):
            continue
        t = re.search(r'\((\.L_x_\d+)\)', rest)
        head = labels.get(t.group(1)) if t else None
        if head is not None and head < addr:
            body = [o for a, o, _ in kernel_ins if head <= a <= addr]
            return {'head': head, 'back_edge': addr, 'bytes': addr + 16 - head, 'instructions': len(body),
                    'ldl': sum(o.startswith('LDL') for o in body), 'stl': sum(o.startswith('STL') for o in body),
                    'conversions': sum(o.startswith(('I2F.F64', 'F2I')) and 'F64' in o for o in body)}
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', default=os.path.join(ROOT, 'nufhe_b200', 'csrc', 'libnufhe_b200.so'))
    ap.add_argument('--kernel', default='blind_rotate_kernelINS_5BrCfgILi2ELi256ELi2ELb1ELb1EEELb0ELb0E',
                    help='substring of the mangled kernel name (default: the gate kernel of the 2-ciphertext shape with '
                         'the FP64 step and a standard key -- its multi-bit instantiation ends in Lb0ELb1E, and a '
                         'shorter default would count both; the NTT one is blind_rotate_kernelINS_5BrCfgILi2ELi256ELi2ELb0ELb0EEELb0E, the '
                         'wide shape blind_rotate_kernelINS_5BrCfgILi1ELi256ELi2ELb0ELb0EEELb0E, the pair shape '
                         'blind_rotate_pair_kernelILb1ELb0E)')
    ap.add_argument('--by-func', action='store_true', help='also split each phase by innermost ff.cuh / br_phases function')
    ap.add_argument('--opcodes', action='store_true', help='per-step histogram of instruction forms (carry-out variants split)')
    ap.add_argument('--json', action='store_true', help='print one JSON object with the per-step totals (used by bench.py)')
    args = ap.parse_args()

    tmp = tempfile.mkdtemp()
    subprocess.check_call(['cuobjdump', '-xelf', 'all', os.path.abspath(args.lib)], cwd=tmp, stdout=subprocess.DEVNULL)
    cubin = [f for f in os.listdir(tmp) if f.endswith('.cubin')][0]
    text = subprocess.run(['nvdisasm', '--print-line-info-inline', '-c', os.path.join(tmp, cubin)],
                          capture_output=True, text=True).stdout.splitlines()

    # phase = line of kernels.cuh inside br2_step
    kpath = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'kernels.cuh')
    ksrc = open(kpath).read().splitlines()
    phase_lines = {}
    in_step = False
    for i, line in enumerate(ksrc, 1):
        if 'void br2_step' in line or 'void br_fft_step' in line:
            in_step = True
        if in_step:
            m = re.search(r'((?:fft_)?phase_[a-z0-9_]+)', line)
            if m:
                phase_lines[i] = m.group(1)
            if line.startswith('}'):
                in_step = False
    step_call_lines = [i for i, l in enumerate(ksrc, 1) if ('br2_step<true' in l or 'br_fft_step<true' in l) and 'void' not in l]
    if 'pair' in args.kernel:
        # the pair shape (blind_rotate_pair_kernel): phases are the pair_* calls of its step loop.  Each pair_* wrapper
        # holds BOTH thread halves (`if (h) f<1>(...) else f<0>(...)`), so a thread executes about half of the static
        # count of a split phase; the MAC loops run twice (two rows per thread).
        phase_lines, in_kernel_src = {}, False
        for i, line in enumerate(ksrc, 1):
            if 'blind_rotate_pair_kernel(' in line:
                in_kernel_src = True
            if in_kernel_src:
                m = re.search(r'\b(pair_[a-z0-9_]+)(?:<[a-z]+>)?\(', line)
                if m:
                    phase_lines[i] = 'phase_' + m.group(1)
                if line.startswith('}'):
                    in_kernel_src = False
        step_call_lines = list(phase_lines)

    # lines of br_phases.cuh inside a `switch (g)` (warp-uniform 4-way): each branch runs for a quarter of the warps
    bpath = os.path.join(ROOT, 'nufhe_b200', 'csrc', 'br_phases.cuh')
    case_lines = {i for i, l in enumerate(open(bpath).read().splitlines(), 1) if re.match(r'\s*(case \d+|default):', l)}

    # lines of br_phases.cuh inside the digit loop of phase_fwd1_both_digits (a real loop, two iterations per step),
    # and inside the output-spectrum loop of the FP64 step's pass 3 (four iterations)
    bsrc0 = open(bpath).read().splitlines()

    def loop_lines(header):
        lines = set()
        for i, l in enumerate(bsrc0, 1):
            if header in l:
                depth, j = 0, i
                while True:
                    depth += bsrc0[j - 1].count('{') - bsrc0[j - 1].count('}')
                    lines.add(j)
                    if depth <= 0 and j > i:
                        break
                    j += 1
        return lines
    twice_lines = loop_lines('for (int j = 0; j < 2; j++)')
    four_lines = loop_lines('for (int s = 0; s < 4; s++)')

    # lines of br_phases.cuh inside an `if (canon_needed(...)) { ... }` block: the rare path of the deferred
    # canonicalisation (taken with probability ~2^-28 per task) -- not part of the executed step
    rare_lines = set()
    bsrc = open(bpath).read().splitlines()
    for i, l in enumerate(bsrc, 1):
        if 'canon_needed(' in l and l.lstrip().startswith('if '):
            depth, j = 0, i
            while True:
                depth += bsrc[j - 1].count('{') - bsrc[j - 1].count('}')
                rare_lines.add(j)
                if depth <= 0 and j > i:
                    break
                if depth <= 0 and '{' not in bsrc[j - 1]:
                    rare_lines.add(j + 1)     # single-statement body on the next line
                    break
                j += 1
            rare_lines.discard(i)             # the test itself is executed

    fn_maps = {}

    def fn_of(path, line):
        if path not in fn_maps:
            fn_maps[path] = enclosing_functions(path)
        return fn_maps[path].get(line)

    in_kernel = False
    chain = []
    counts = collections.defaultdict(lambda: collections.Counter())
    byfunc = collections.defaultdict(lambda: collections.Counter())
    rx_line = re.compile(r'//## File "([^"]+)", line (\d+)')
    rx_ins = re.compile(r'^\s+/\*([0-9a-f]+)\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)(.*)')
    forms = collections.Counter()
    loop_addrs = []           # addresses of the instructions of the rotating step loop's phases
    kernel_ins = []           # (address, opcode, operands) of every instruction of the kernel
    labels, pending_labels = {}, []
    rx_label = re.compile(r'^(\.L_x_\d+):')
    for ln in text:
        if ln.startswith('.text.'):
            in_kernel = args.kernel in ln
            chain = []
            continue
        if not in_kernel:
            continue
        m = rx_line.search(ln)
        if m:
            if not chain or chain_done:
                chain = []
                chain_done = False
            chain.append((m.group(1), int(m.group(2))))
            continue
        m = rx_label.match(ln)
        if m:
            pending_labels.append(m.group(1))
            continue
        m = rx_ins.match(ln)
        if not m:
            continue
        chain_done = True
        addr, op, rest = int(m.group(1), 16), m.group(2), m.group(3)
        kernel_ins.append((addr, op, rest))
        for lab in pending_labels:
            labels[lab] = addr
        pending_labels = []
        pipe = pipe_of(op)
        phase = 'other'
        in_loop = False
        for path, line in chain:
            if path.endswith('kernels.cuh'):
                if line in phase_lines:
                    phase = phase_lines[line]
                if line in step_call_lines:
                    in_loop = True
        if phase != 'other' and not in_loop:
            phase = 'plain:' + phase     # the non-rotating instantiation (nb_external_product)
        if in_loop and phase != 'other':
            loop_addrs.append(addr)
        w = 0.25 if any(path.endswith('br_phases.cuh') and line in case_lines for path, line in chain) else 1
        if any(path.endswith('br_phases.cuh') and line in twice_lines for path, line in chain):
            w *= 2
        if any(path.endswith('br_phases.cuh') and line in four_lines for path, line in chain):
            w *= 4
        if any(path.endswith('br_phases.cuh') and line in rare_lines for path, line in chain):
            counts['rare:' + phase][pipe] += w
            continue
        counts[phase][pipe] += w
        if args.opcodes and phase.startswith(('phase_', 'fft_phase_')):
            forms[instruction_form(op, rest)] += w * (
                1 if ('BrCfgILi1E' in args.kernel and phase.startswith('phase_fwd')) else STEP_MULT.get(phase, 1))
        if args.by_func and chain:
            inner = None
            for path, line in chain:
                f = fn_of(path, line)
                if f and (path.endswith('ff.cuh')):
                    inner = f
                    break
            if inner is None:
                inner = fn_of(*chain[0]) or '?'
            byfunc[phase][(inner, pipe)] += w

    # the wide shape (1 ciphertext on 256 threads) runs the forward phases in one sweep
    mult = dict(STEP_MULT, phase_fwd1=1, phase_fwd2=1, phase_fwd3=1) if 'BrCfgILi1E' in args.kernel else STEP_MULT
    loop = step_loop(kernel_ins, loop_addrs, labels)
    if args.json:
        import json
        tot = collections.Counter()
        for phase, c in counts.items():
            if phase.startswith(('phase_', 'fft_phase_')):
                for k, v in c.items():
                    tot[k] += v * mult.get(phase, 1)
        print(json.dumps({'kernel': args.kernel, 'per_thread_step': {k: tot[k] for k in ('alu', 'fma', 'fp64', 'lsu', 'uni', 'other')},
                          'per_thread_step_total': sum(tot.values()),
                          'phases': {ph: sum(c.values()) * mult.get(ph, 1) for ph, c in counts.items() if ph.startswith(('phase_', 'fft_phase_'))},
                          'step_loop': loop}))
        return 0
    print('%-22s %7s %7s %7s %7s %7s %7s %8s' % ('phase (static)', 'alu', 'fma', 'fp64', 'lsu', 'uni', 'other', 'total'))
    tot = collections.Counter()
    for phase in sorted(counts):
        c = counts[phase]
        print('%-22s %7d %7d %7d %7d %7d %7d %8d' % (phase, c['alu'], c['fma'], c['fp64'], c['lsu'], c['uni'], c['other'], sum(c.values())))
        if phase.startswith(('phase_', 'fft_phase_')):
            for k, v in c.items():
                tot[k] += v * mult.get(phase, 1)
    print('%-22s %7d %7d %7d %7d %7d %7d %8d   (sweeps, MAC rows and switch weights applied)' % (
        'per step, per thread', tot['alu'], tot['fma'], tot['fp64'], tot['lsu'], tot['uni'], tot['other'], sum(tot.values())))
    if loop:
        print('step loop: %#x - back-edge %#x, %d bytes (%d instructions); static in the loop: %d LDL, %d STL (spill), '
              '%d I2F.F64 / F2I.F64 (conversion)' % (loop['head'], loop['back_edge'], loop['bytes'], loop['instructions'],
                                                       loop['ldl'], loop['stl'], loop['conversions']))
    if args.opcodes:
        # issue cost in SMSP cycles per warp-instruction (tools/microbench/pipes.cu): 2 on either integer
        # pipe, except IMAD.WIDE with a 64-bit addend: 4
        alu_c = sum(2 * v for k, v in forms.items() if pipe_of(k.split('(')[0]) == 'alu')
        fma_c = sum((COST.get(k.replace('.P', ''), 2)) * v for k, v in forms.items() if pipe_of(k.split('(')[0]) == 'fma')
        print('-- pipe cycles per step, per warp: ALU %.0f  FMA %.0f  (sum %.0f, balanced bound %.0f)' % (
            alu_c, fma_c, alu_c + fma_c, (alu_c + fma_c) / 2))
        print('-- instruction forms per step, per thread')
        for k, v in sorted(forms.items(), key=lambda kv: -kv[1]):
            if v >= 4:
                print('   %-20s %7.0f' % (k, v))
    if args.by_func:
        for phase in sorted(byfunc):
            if not phase.startswith(('phase_', 'fft_phase_')):
                continue
            print('--', phase)
            agg = collections.defaultdict(collections.Counter)
            for (fn, pipe), v in byfunc[phase].items():
                agg[fn][pipe] += v
            for fn, c in sorted(agg.items(), key=lambda kv: -sum(kv[1].values())):
                print('   %-24s alu %6d  fma %6d  lsu %5d  other %5d' % (fn, c['alu'], c['fma'], c['lsu'], c['uni'] + c['other']))


if __name__ == '__main__':
    sys.exit(main())
