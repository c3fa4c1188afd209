#!/usr/bin/env python
"""Constructor signatures of the reference's implicit-solvent and toluene test systems (build container only): argument
names and default-value source text, read from the reference's AST.  Output: tests/golden/implicit_signatures_golden.json"""
import ast, json, os

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/openmmtools/testsystems.py'
CLASSES = ['AlanineDipeptideImplicit', 'TolueneVacuum', 'TolueneImplicit', 'TolueneImplicitHCT', 'TolueneImplicitOBC1',
           'TolueneImplicitOBC2', 'TolueneImplicitGBn', 'TolueneImplicitGBn2']
tree = ast.parse(open(REF).read())
out = {}
for name in CLASSES:
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == name][0]
    a = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == '__init__'][0].args
    names = [x.arg for x in a.args]
    defaults = [None] * (len(names) - len(a.defaults)) + [ast.unparse(d) for d in a.defaults]
    out[name] = {'args': [[n, d] for n, d in zip(names, defaults) if n != 'self'], 'kwarg': a.kwarg.arg if a.kwarg else None}
dst = os.path.join(HERE, 'implicit_signatures_golden.json')
json.dump(out, open(dst, 'w'), indent=1, sort_keys=True)
print('wrote', dst, len(out))
