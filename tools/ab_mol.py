"""A/B check of molecule-kernel builds on one GPU (development aid).
  python tools/ab_mol.py libA.so libB.so ...     each library runs in its own process (RX_B200_LIB, 'default' = the library
  of this tree), alternated AB_ROUNDS times (default 1).  Cases: every molecule of tests/test_gpu_molecule.py's MOLECULES in
  vacuum and every system of tests/test_gpu_implicit.py's SYSTEMS with OBC1 and OBC2.  For each case it prints digests of
  compute_energies() on perturbed positions, of the positions, velocities and replica energies after a 50-step launch, and
  of the minimiser's rms, iterations and positions; all builds must print the same energy and launch digests.  The first
  library's minimised positions are the reference of a max |dx| printed for the others.  Then it times minimize() on
  alanine dipeptide in vacuum and in OBC1 implicit solvent at K = 128 (AB_MIN_REPS calls each, default 3).  AB_CASES (e.g.
  'vacuum:decane,OBC2:toluene') selects cases; AB_OUT is where the minimised positions go (default build/ab_mol)."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.environ.get('AB_OUT', os.path.join(ROOT, 'build', 'ab_mol'))

CHILD = r'''
import sys, os, time, zlib
sys.path.insert(0, %r)
sys.path.insert(0, os.path.join(%r, 'tests'))
import numpy as np
import implicit_helpers as IH
from test_gpu_molecule import MOLECULES, make_engine
from test_gpu_implicit import SYSTEMS
out, tag = sys.argv[1], sys.argv[2]
dig = lambda *a: '%%08x' %% zlib.crc32(b''.join(np.ascontiguousarray(v).tobytes() for v in a))
cases = [('vacuum', k) for k in MOLECULES] + [(m, k) for m in ('OBC1', 'OBC2') for k in SYSTEMS]
sel = os.environ.get('AB_CASES')
if sel:
    cases = [tuple(c.split(':')) for c in sel.split(',')]
mins = {}
for model, name in cases:
    if model == 'vacuum':
        system, x = MOLECULES[name]()
    else:
        system, x = SYSTEMS[name]()
        system = IH.with_model(system, model)
    temps = np.array([300.0, 350.0, 420.0, 600.0])
    K = len(temps)
    rng = np.random.default_rng(3)
    xs = np.stack([x + rng.normal(0, 0.004, x.shape) for _ in temps])
    e = make_engine(system, temps)
    e.set_positions(xs)
    d_u = dig(e.compute_energies())
    e.set_integrator(0.002, 5.0, 50, 'V R O R V')
    e.set_positions(np.stack([x] * K)); e.randomize_velocities(11)
    e.propagate(5, 1)
    xl = e.get_positions()
    d_l = dig(xl, e.get_velocities(), *e.get_replica_energies())
    rms, its = e.minimize(5.0, max_iterations=2000)
    xm = e.get_positions()
    e.close()
    mins['%%s:%%s' %% (model, name)] = xm
    print('%%-36s energies %%s  launch %%s  minimiser rms %%s its %%s x %%s  (its %%s)' %% (
        model + ':' + name, d_u, d_l, dig(rms), dig(its), dig(xm), its.tolist()))
    sys.stdout.flush()
np.savez(os.path.join(out, tag + '.npz'), **mins)
for model, sysf in (('vacuum', lambda: MOLECULES['alanine-dipeptide']()), ('OBC1', lambda: SYSTEMS['alanine-dipeptide']())):
    system, x = sysf()
    K = 128
    temps = np.linspace(300.0, 600.0, K)
    e = make_engine(system, temps)
    e.set_integrator(0.002, 5.0, 200, 'V R O R V')
    e.set_positions(np.stack([x] * K)); e.randomize_velocities(5)
    e.propagate(9, 1)
    x0 = e.get_positions()
    ms = []
    for rep in range(int(os.environ.get('AB_MIN_REPS', '3'))):
        e.set_positions(x0)
        t0 = time.perf_counter(); rms, its = e.minimize(5.0, max_iterations=5000); ms.append(1e3 * (time.perf_counter() - t0))
    e.close()
    print('minimize() %%-6s K=128: %%s ms per call; iterations max %%d mean %%.1f; rms digest %%s' %% (
        model, ' '.join('%%.1f' %% t for t in ms), its.max(), its.mean(), dig(rms, its)))
    sys.stdout.flush()
''' % (ROOT, ROOT)

os.makedirs(OUT, exist_ok=True)
try:
    print('card:', subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                                  text=True).stdout.strip().splitlines()[0])
except (OSError, IndexError):
    print('card: unknown')
libs = sys.argv[1:]
for rnd in range(int(os.environ.get('AB_ROUNDS', '1'))):
    for n, lib in enumerate(libs):
        env = dict(os.environ)
        if lib != 'default':
            env['RX_B200_LIB'] = os.path.abspath(lib)
        print('== round %d  %s' % (rnd, lib))
        try:
            r = subprocess.run([sys.executable, '-c', CHILD, OUT, 'r%d_lib%d' % (rnd, n)], env=env, capture_output=True, text=True,
                               timeout=int(os.environ.get('AB_TIMEOUT', '1200')))
            print(r.stdout.rstrip() if r.returncode == 0 else (r.stdout + r.stderr)[-3000:])
        except subprocess.TimeoutExpired:
            print('TIMEOUT')
        sys.stdout.flush()

import numpy as np
ref = os.path.join(OUT, 'r0_lib0.npz')
if os.path.exists(ref):
    a = np.load(ref)
    for n in range(1, len(libs)):
        p = os.path.join(OUT, 'r0_lib%d.npz' % n)
        if not os.path.exists(p):
            continue
        b = np.load(p)
        print('== minimised positions, %s against %s: max |dx| in nm' % (libs[n], libs[0]))
        for k in a.files:
            print('  %-36s %.3e' % (k, np.abs(a[k] - b[k]).max()))
