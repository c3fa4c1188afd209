#!/usr/bin/env python
"""Parameter fixtures of the implicit-solvent test systems, parsed from AMBER files by openmmtools_b200.amber (copies kept
next to this script) and stored as plain numbers, so that the package needs no AMBER files at run time:
  * AlanineDipeptideImplicit: the GB radii (nm) and screening factors of alanine-dipeptide.prmtop (the rest of its
    force field is alanine_dipeptide_vacuum.json, made by make_aladip_fixture.py);
  * TolueneVacuum / TolueneImplicit*: the whole force field and positions of benzene-toluene-implicit/solvent.{prmtop,inpcrd}
    (toluene-solvent.{prmtop,inpcrd} here) plus its GB radii and screening factors.
Output: openmmtools_b200/data/alanine_dipeptide_implicit.json, openmmtools_b200/data/toluene_implicit.json"""
import json, os, sys
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
from openmmtools_b200 import amber


def gb(d):
    return dict(radii=[float(v) for v in d['radii']], screen=[float(v) for v in d['screen']], radius_set=d['radius_set'])


def build():
    aladip = gb(amber.read_prmtop(os.path.join(HERE, 'alanine-dipeptide.prmtop')))
    d = amber.read_prmtop(os.path.join(HERE, 'toluene-solvent.prmtop'))
    x = amber.read_inpcrd(os.path.join(HERE, 'toluene-solvent.inpcrd'))
    toluene = dict(names=d['names'], mass=[float(v) for v in d['mass']], charge=[float(v) for v in d['charge']],
                   sigma=[float(v) for v in d['sigma']], epsilon=[float(v) for v in d['epsilon']],
                   bonds=[[int(b[0]), int(b[1]), float(b[2]), float(b[3]), bool(b[4])] for b in d['bonds']],
                   angles=[[int(a[0]), int(a[1]), int(a[2]), float(a[3]), float(a[4])] for a in d['angles']],
                   torsions=[[int(t[0]), int(t[1]), int(t[2]), int(t[3]), int(t[4]), float(t[5]), float(t[6])] for t in d['torsions']],
                   exclusions=[[int(i), int(j)] for i, j in d['exclusions']],
                   exceptions=[[int(e[0]), int(e[1]), float(e[2]), float(e[3]), float(e[4])] for e in d['exceptions']],
                   positions=[[float(c) for c in r] for r in x], **gb(d))
    return aladip, toluene


if __name__ == '__main__':
    data = os.path.join(HERE, '..', '..', 'openmmtools_b200', 'data')
    for name, d in zip(('alanine_dipeptide_implicit.json', 'toluene_implicit.json'), build()):
        dst = os.path.join(data, name)
        json.dump(d, open(dst, 'w'))
        print('wrote', os.path.abspath(dst), os.path.getsize(dst))
