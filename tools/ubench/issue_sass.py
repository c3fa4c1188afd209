"""Opcode histogram of the timed loop of every case of tools/ubench/issue.cu (the largest backward-branch body of each
k_issue<C> instantiation), to check that a case's loop holds the intended opcode and otherwise only its counter and
branch.  Usage: python tools/ubench/issue_sass.py tools/ubench/issue"""
import collections, re, subprocess, sys


def loops(path):
    out = subprocess.run(['cuobjdump', '-sass', path], capture_output=True, text=True).stdout.splitlines()
    fns, cur = {}, None
    for line in out:
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = fns.setdefault(m.group(1), [])
            continue
        m = re.match(r'\s*/\*([0-9a-f]{4,})\*/\s+(.*?);', line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2).strip()))
    for fn, ins in fns.items():
        m = re.search(r'k_issueILi(\d+)E', fn)
        if not m:
            continue
        best = None
        for a, t in ins:
            b = re.search(r'BRA\s+(?:\w+,\s*)?0x([0-9a-f]+)', t)
            if b and int(b.group(1), 16) < a and (best is None or a - int(b.group(1), 16) > best[1] - best[0]):
                best = (int(b.group(1), 16), a)
        if best is None:
            continue
        hist = collections.Counter()
        for a, t in ins:
            if best[0] <= a <= best[1]:
                f = t.split()
                hist[(f[1] if f[0].startswith('@') else f[0]).split('.')[0]] += 1
        yield int(m.group(1)), hist


if __name__ == '__main__':
    for c, hist in sorted(loops(sys.argv[1])):
        print('case %2d: %s' % (c, '  '.join('%s %d' % kv for kv in hist.most_common())))
