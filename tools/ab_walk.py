"""A/B timing of the swap-all walker builds on one GPU (development aid).
  python tools/ab_walk.py libA.so libB.so ...     each library runs in its own process (RX_B200_LIB, 'default' = the
  library of this tree), alternated AB_ROUNDS times (default 3).  Cases: K = 256 on the real alchemical-LJ energy matrix
  tools/data/u_lj_256.npy (K^3 attempts: k_mix_walk2 + k_mix_walk_pow2<true>), and the 'ladder' and 'flat' matrices of
  tests/golden/energy_models.py with AB_NSWAP attempts (default 2 000 000) at K = 100, 200 (k_mix_walk2c), 300, 500, 1000
  (k_mix_walk_cand), 512, 1024 (k_mix_walk_pow2<false>), with RX_NO_FILTER=1 at K = 64 and 256 (k_mix_walk_pow2<false>) and,
  with RX_WALK_SERIAL=1, at K = 300 (k_mix_walk_serial alone).  AB_CASES (e.g. 'lj:256,ladder:300,flat:64:nofilter,
  ladder:300:serial') selects cases.  Every case makes AB_REPS (default 3) calls in one engine and prints walker ms per call,
  the mix_stats of the last call, a permutation / count-matrix digest of every call and the launches of all calls by phase
  (mix, propagate, energies, stream generation): all builds must print the same statistics, digests and launches."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DEFAULT_CASES = ('lj:256,ladder:100,flat:200,ladder:300,flat:300,ladder:500,flat:500,ladder:1000,flat:1000,ladder:512,'
                 'flat:512,ladder:1024,flat:1024,ladder:64:nofilter,flat:64:nofilter,ladder:256:nofilter,flat:256:nofilter,'
                 'ladder:300:serial')

CHILD = r'''
import sys, os, zlib
sys.path.insert(0, %r)
sys.path.insert(0, os.path.join(%r, 'tests', 'golden'))
import numpy as np
from energy_models import energies
from openmmtools_b200._engine import Engine
for case in os.environ.get('AB_CASES', %r).split(','):
    f = case.split(':')
    model, K = f[0], int(f[1])
    if 'nofilter' in f[2:]: os.environ['RX_NO_FILTER'] = '1'
    else: os.environ.pop('RX_NO_FILTER', None)
    if 'serial' in f[2:]: os.environ['RX_WALK_SERIAL'] = '1'
    else: os.environ.pop('RX_WALK_SERIAL', None)
    if model == 'lj':
        u = np.load(os.path.join(%r, 'tools', 'data', 'u_lj_256.npy'))[:K, :K].copy()
        nswap = K ** 3
    else:
        u = energies(model, K, 4242 + K)
        nswap = int(os.environ.get('AB_NSWAP', '2000000'))
    e = Engine(0, K, K, 0)
    e.set_energies(u); e.set_replica_states(np.arange(K)); e.mix_seed(1234, 0)
    ms_list, dig = [], []
    for rep in range(int(os.environ.get('AB_REPS', '3'))):
        st, nacc, nprop = e.mix_swap_all(nswap)
        ms = e.mix_stats()
        ms_list.append(ms['walker_ms'])
        dig.append('%%08x/%%08x' %% (zlib.crc32(st.tobytes()), zlib.crc32(nacc.tobytes()) ^ zlib.crc32(nprop.tobytes())))
    launches = e.phase_times()['launches_by_phase']
    e.close()
    print('%%-22s walker ms %%s  rounds %%d exact_exp %%d passes %%d words %%d  digests %%s  launches %%s' %% (
        case, ' '.join('%%8.2f' %% m for m in ms_list), ms['rounds'], ms['exact_exp'], ms['passes'], ms['words'], ' '.join(dig),
        launches))
    sys.stdout.flush()
''' % (ROOT, ROOT, DEFAULT_CASES, ROOT)

for rnd in range(int(os.environ.get('AB_ROUNDS', '3'))):
    for lib in sys.argv[1:]:
        env = dict(os.environ)
        if lib != 'default':
            env['RX_B200_LIB'] = os.path.abspath(lib)
        print('== round %d  %s' % (rnd, lib))
        try:
            r = subprocess.run([sys.executable, '-c', CHILD], env=env, capture_output=True, text=True,
                               timeout=int(os.environ.get('AB_TIMEOUT', '900')))
            print(r.stdout.rstrip() if r.returncode == 0 else (r.stdout + r.stderr)[-2000:])
        except subprocess.TimeoutExpired:
            print('TIMEOUT')
        sys.stdout.flush()
