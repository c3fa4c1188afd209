"""Compare the kernels of two builds of librx_b200.so (or of two objects) function by function.

For every function `cuobjdump -sass` prints, it reports registers and stack frame (`cuobjdump -res-usage`) on both
sides and whether the code is byte-identical, identical once constant-bank operands c[0x0][0x...] are masked (a
parameter struct changed layout), or different (with the change in instruction count).  Functions are matched by name
and template arguments, so a kernel whose parameter list changed is still compared; functions present on one side only
are listed.  Used to check that a refactor keeps the SASS of the kernels it touches.
Usage: python tools/sass_diff.py <old.so> <new.so> [name-regex]"""
import re, subprocess, sys

INS = re.compile(r'\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;\s*/\* (0x[0-9a-f]{16}) \*/')
ENC = re.compile(r'\s*/\* (0x[0-9a-f]{16}) \*/\s*$')
CBANK = re.compile(r'c\[0x0\]\[0x[0-9a-f]+\]')
BRANCH = re.compile(r'\b(BRA|BRX|CALL\.REL(\.NOINC)?|BSSY|JMP|BREAK|SSY)\b.*?0x[0-9a-f]+')


def demangle(names):
    """One c++filt call for all names."""
    out = subprocess.run(['c++filt'], input='\n'.join(names), capture_output=True, text=True, check=True).stdout
    return out.splitlines()


def keys(names):
    """mangled -> key: the demangled name without its parameter list (`k_propagate<true, false, 1, false, false, false>`),
    so that a kernel whose parameters changed is still matched; the full demangled name where that would be ambiguous"""
    full = demangle(names)
    short = [d.split('(', 1)[0].removeprefix('void ') for d in full]
    return {n: (s if short.count(s) == 1 else d) for n, s, d in zip(names, short, full)}


def sass(path):
    """key -> (instruction texts, encodings)"""
    out = subprocess.run(['cuobjdump', '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = funcs.setdefault(m.group(1), ([], []))
            continue
        if cur is None:
            continue
        m = INS.match(line)
        if m:
            cur[0].append(m.group(1))
            cur[1].append(m.group(2))
            continue
        m = ENC.match(line)
        if m and cur[1]:
            cur[1][-1] += m.group(1)
    k = keys(list(funcs))
    return {k[n]: v for n, v in funcs.items()}


def res_usage(path):
    out = subprocess.run(['cuobjdump', '-res-usage', path], capture_output=True, text=True, check=True).stdout
    found = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r'Function (\S+):\s*REG:(\d+) STACK:(\d+)', out)}
    k = keys(list(found))
    return {k[n]: v for n, v in found.items()}


def masked(texts):
    # constant-bank offsets move with the parameter layout; branch targets move with any change of length before them
    return [BRANCH.sub(lambda m: m.group(0).rsplit('0x', 1)[0] + '0x*', CBANK.sub('c[0x0][*]', t)) for t in texts]


def main():
    old_path, new_path = sys.argv[1], sys.argv[2]
    pat = re.compile(sys.argv[3] if len(sys.argv) > 3 else '')
    old, new = sass(old_path), sass(new_path)
    ru_old, ru_new = res_usage(old_path), res_usage(new_path)
    for n in sorted(set(old) - set(new)):
        if pat.search(n): print(f'only in old  {n}')
    for n in sorted(set(new) - set(old)):
        if pat.search(n): print(f'only in new  {n}')
    worse = 0
    for n in sorted(set(old) & set(new)):
        if not pat.search(n):
            continue
        (to, eo), (tn, en) = old[n], new[n]
        if eo == en:
            kind = 'identical'
        elif masked(to) == masked(tn):
            kind = 'same-masked'
        else:
            kind = f'differs {len(tn) - len(to):+d} of {len(to)}'
        ro, rn = ru_old.get(n, (-1, -1)), ru_new.get(n, (-1, -1))
        flag = ''
        if rn[0] != ro[0] or rn[1] > ro[1]:
            flag = '  <-- resources'
            worse += 1
        print(f'{kind:24s} REG {ro[0]:3d}->{rn[0]:3d} STACK {ro[1]:4d}->{rn[1]:4d}  {n}{flag}')
    return 1 if worse else 0


if __name__ == '__main__':
    sys.exit(main())
