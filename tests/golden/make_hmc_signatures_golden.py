#!/usr/bin/env python
"""Signatures of the reference's HMCMove (build container only): argument names and default-value source text of
__init__, and the keys __getstate__ adds, read from the reference's AST.  Output: tests/golden/hmc_signatures_golden.json"""
import ast, json, os

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/openmmtools/mcmc.py'
tree = ast.parse(open(REF).read())
cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == 'HMCMove'][0]
fns = {n.name: n for n in cls.body if isinstance(n, ast.FunctionDef)}
a = fns['__init__'].args
names = [x.arg for x in a.args]
defaults = [None] * (len(names) - len(a.defaults)) + [ast.unparse(d) for d in a.defaults]
keys = sorted({t.slice.value for n in ast.walk(fns['__getstate__']) if isinstance(n, ast.Assign) for t in n.targets
               if isinstance(t, ast.Subscript) and isinstance(t.slice, ast.Constant)})
out = {'mcmc.py:HMCMove.__init__': {'args': [[n, d] for n, d in zip(names, defaults) if n != 'self'],
                                    'kwarg': a.kwarg.arg if a.kwarg else None, 'line': fns['__init__'].lineno},
       'mcmc.py:HMCMove.__getstate__': {'keys': keys}}
dst = os.path.join(HERE, 'hmc_signatures_golden.json')
json.dump(out, open(dst, 'w'), indent=1, sort_keys=True)
print('wrote', dst, out)
