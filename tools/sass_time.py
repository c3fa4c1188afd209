"""Static single-warp timing of a straight-line SASS path: stall counts and scoreboards from the control bits (assumed
variable latencies), plus what a LONE warp can issue: every instruction holds the warp's issue port for HOLD cycles and its
pipe for BUSY cycles, and issues at max(T, scoreboards, busy[pipe]).
Usage: python tools/sass_time.py obj fn seg[,seg...]  with seg = start-end (hex)

The issue table was measured with tools/ubench/issue.cu (streams of 8 independent chains, one warp; the three exited
helper warps of a 128-thread block change nothing) on one NVIDIA H100 80GB HBM3, 700 W power limit, 1980 MHz,
2026-10-16, loop overhead (14 cycles per 32 instructions, from the FADD stream) removed:
  ALU pipe (LOP3 SHF IADD3 ISETP SEL PRMT FSETP FMNMX ..)  2.0 cycles each, and 2 + 1 beside an FFMA or IMAD: the warp's
      issue is held for both cycles (a 16-lane pipe takes a warp in two halves)
  FP32 (FADD FFMA FMUL)   1.0;   IMAD 2.0 alone, 1 beside ALU instructions (holds the issue port one cycle, its pipe two)
  uniform datapath        ULOP3 USHF 2.4, UIADD3 UPOPC 2.0 alone; beside vector instructions about 0.5 cycles of issue
  VOTE 2.0   SHFL 3.9   POPC 7.7
  LDS (any width, conflict free) 4.2, 3.7 of them holding the issue port;  STS.64 5.9;  LDGSTS (cp.async 16 B) 14
(not reproduced: FFMA interleaved with IMAD measured 3.8 cycles per pair, the table gives 3.)"""
import sys
sys.path.insert(0, __file__.rsplit('/', 1)[0])
from sass_ctl import decode

LAT = {'LDS': 30, 'LDG': 300, 'POPC': 14, 'LDC': 40, 'LDCU': 40, 'S2UR': 30, 'SHFL': 26, 'MUFU': 18, 'STS': 12, 'STG': 12,
       'F2F': 14, 'I2F': 14, 'ATOMS': 40, 'BAR': 30, 'MEMBAR': 40, 'S2R': 30, 'LDSM': 30, 'REDUX': 20}
RLAT = 8

# opcode -> pipe
PIPE = {}
for _p, _ops in {
    'alu': 'LOP3 SHF IADD3 ISETP SEL PRMT FSETP FMNMX FSEL LEA VIADD VIMNMX VIMNMX3 IMNMX PLOP3 P2R R2P MOV IABS BMSK SGXT '
           'VOTE CS2R FCHK',
    'fp32': 'FADD FFMA FMUL HFMA2 HADD2 HMUL2',
    'imad': 'IMAD',
    'uni': 'ULOP3 USHF UIADD3 UPOPC UMOV UISETP ULEA UIMAD USEL UPRMT UFLO UPLOP3 VOTEU R2UR UP2UR UR2UP',
    'lsu': 'LDS STS LDG STG LDGSTS ATOMS ATOMG LDSM LD ST LDL STL RED SHFL',
    'xu': 'POPC MUFU F2F I2F F2I FLO BREV I2FP F2FP',
    'f64': 'DADD DMUL DFMA DSETP',
    'ctl': 'BRA EXIT NOP DEPBAR LDGDEPBAR BAR WARPSYNC BSSY BSYNC S2R S2UR LDC LDCU ULDC CALL RET MEMBAR ERRBAR YIELD '
           'NANOSLEEP REDUX MATCH BREAK BMOV',
}.items():
    for _o in _ops.split():
        PIPE[_o] = _p

# pipe -> (cycles the issue port is held, cycles the pipe is busy); per-opcode exceptions below
ISSUE = {'alu': (2.0, 2.0), 'fp32': (1.0, 1.0), 'imad': (1.0, 2.0), 'uni': (0.5, 2.4), 'lsu': (3.7, 4.2), 'xu': (1.0, 7.7),
         'f64': (2.0, 2.0), 'ctl': (1.0, 1.0)}
ISSUE_OP = {'UIADD3': (0.5, 2.0), 'UPOPC': (0.5, 2.0), 'STS': (5.4, 5.9), 'STG': (5.4, 5.9), 'LDGSTS': (13.5, 14.0),
            'SHFL': (3.4, 3.9)}


def opcode(text):
    f = text.split()
    return (f[1] if f[0].startswith('@') else f[0]).split('.')[0]


def pipe_of(text):
    """The pipe of one SASS instruction; an opcode that is not in the table is an error, not a default."""
    op = opcode(text)
    if op not in PIPE:
        raise KeyError('sass_time: no pipe for opcode %s (%s)' % (op, text))
    return PIPE[op]


def issue_of(text):
    op = opcode(text)
    if '@!PT' in text.split()[0]:          # never executed (alignment filler of the compiler): one issue slot
        return 'ctl', (1.0, 1.0)
    p = pipe_of(text)
    return p, ISSUE_OP.get(op, ISSUE[p])


def schedule(seq, verbose=False, pipes=True):
    """Time a list of instructions (dicts: text, stall, wait, wbar, rbar; addr optional).  Returns (total cycles, cycles
    of pipe occupancy per pipe).  pipes=False is the model without issue costs (stall counts and scoreboards alone)."""
    T = 0.0
    sb = [0.0] * 6
    busy = {}
    total = {}
    for i in seq:
        arm = max([sb[s] for s in range(6) if (i['wait'] >> s) & 1] or [0])
        T0 = T
        T = max(T, arm)
        pipe, (hold, occ) = issue_of(i['text'])
        if pipes:
            T = max(T, busy.get(pipe, 0.0))
            busy[pipe] = T + occ
        total[pipe] = total.get(pipe, 0.0) + occ
        base = opcode(i['text'])
        if i['wbar'] < 6:
            sb[i['wbar']] = max(sb[i['wbar']], T + LAT.get(base, 30))
        if i['rbar'] < 6:
            sb[i['rbar']] = max(sb[i['rbar']], T + RLAT)
        if verbose:
            print('%7.1f %s%05x st=%2d %-4s %s' % (T, '*' if T > T0 else ' ', i.get('addr', 0), i['stall'], pipe, i['text']))
        # (a stall count of 1 is the encoding's minimum, not a constraint: the issue table says what the slot costs)
        T += max(i['stall'], 1) if not pipes else (hold if i['stall'] <= 1 else max(i['stall'], hold))
    return T, total


def ins(text, stall=1, wait=0, wbar=7, rbar=7):
    """A hand-made instruction for schedule()."""
    return dict(text=text, stall=stall, wait=wait, wbar=wbar, rbar=rbar)


def run(code, segs, verbose=True, pipes=True):
    by = {i['addr']: k for k, i in enumerate(code)}
    seq = []
    for a, b in segs:
        k = by[a]
        while code[k]['addr'] <= b:
            seq.append(code[k])
            k += 1
    return schedule(seq, verbose, pipes)


if __name__ == '__main__':
    code = decode(sys.argv[1], sys.argv[2])
    segs = [tuple(int(x, 16) for x in s.split('-')) for s in sys.argv[3].split(',')]
    T, total = run(code, segs)
    print('pipe occupancy', '  '.join('%s %.0f' % kv for kv in sorted(total.items())))
    print('total', round(T), ' (stall counts and scoreboards alone: %d)' % run(code, segs, False, False)[0])
