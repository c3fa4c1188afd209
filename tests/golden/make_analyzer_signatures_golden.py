#!/usr/bin/env python
"""Constructor signatures of the reference's MultiStateSamplerAnalyzer and ReplicaExchangeAnalyzer (build container
only): the positional arguments of PhaseAnalyzer.__init__ (which MultiStateSamplerAnalyzer.__init__ forwards through
*args / **kwargs) followed by MultiStateSamplerAnalyzer's keyword-only arguments, names and default-value source text,
read from the reference's AST.  Output: tests/golden/analyzer_signatures_golden.json"""
import ast, json, os

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/openmmtools/multistate/'


def init_of(path, cls_name):
    tree = ast.parse(open(REF + path).read())
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name][0]
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == '__init__']
    return cls, (fns[0] if fns else None)


_, base = init_of('multistateanalyzer.py', 'PhaseAnalyzer')
_, msa = init_of('multistateanalyzer.py', 'MultiStateSamplerAnalyzer')
rex, rex_init = init_of('replicaexchange.py', 'ReplicaExchangeAnalyzer')
assert rex_init is None and [b.id for b in rex.bases] == ['MultiStateSamplerAnalyzer']
a = base.args
names = [x.arg for x in a.args]
defaults = [None] * (len(names) - len(a.defaults)) + [ast.unparse(d) for d in a.defaults]
args = [[n, d] for n, d in zip(names, defaults) if n != 'self']
kwonly = [[x.arg, None if d is None else ast.unparse(d)] for x, d in zip(msa.args.kwonlyargs, msa.args.kw_defaults)]
entry = {'args': args, 'kwonly': kwonly, 'line': msa.lineno}
out = {'multistate/multistateanalyzer.py:MultiStateSamplerAnalyzer.__init__': entry,
       'multistate/replicaexchange.py:ReplicaExchangeAnalyzer.__init__': entry}
dst = os.path.join(HERE, 'analyzer_signatures_golden.json')
json.dump(out, open(dst, 'w'), indent=1, sort_keys=True)
print('wrote', dst, out)
