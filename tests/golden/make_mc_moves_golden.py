#!/usr/bin/env python
"""Golden data for the Monte Carlo rigid-body moves, from the REAL reference code (build container only).

``MCDisplacementMove.displace_positions``, ``MCRotationMove._generate_uniform_quaternion``,
``_rotation_matrix_from_quaternion``, ``rotate_positions`` and ``MetropolizedMove.apply`` are lifted by AST from
/root/reference/openmmtools/mcmc.py and run with injected ``np.random.randn`` / ``np.random.rand`` draws; ``apply`` runs on
stand-ins for the context cache, the sampler state and the thermodynamic state, which hand it given reduced energies.
The constructor signatures of the four classes and the keys of their ``__getstate__`` are recorded as well.

Output: tests/golden/mc_moves_golden.npz
"""
import ast, json, os, sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from openmmtools_b200 import unit as u

REF = '/root/reference/openmmtools/mcmc.py'
TREE = ast.parse(open(REF).read())
CLASSES = {n.name: n for n in TREE.body if isinstance(n, ast.ClassDef)}


class _Draws:
    """np.random stand-in: randn / rand return the queued arrays."""

    def __init__(self):
        self.queue = []

    def randn(self, n):
        return np.asarray(self.queue.pop(0), np.float64)[:n]

    def rand(self, n=None):
        v = np.asarray(self.queue.pop(0), np.float64)
        return float(v[0]) if n is None else v[:n]


class _NP:
    def __init__(self, draws):
        self.random = draws

    def __getattr__(self, name):
        return getattr(np, name)


DRAWS = _Draws()
NS = {'np': _NP(DRAWS), 'unit': u, 'copy': __import__('copy')}


def lift(cls, name):
    fn = [n for n in CLASSES[cls].body if isinstance(n, ast.FunctionDef) and n.name == name][0]
    fn.decorator_list = []
    mod = ast.Module(body=[fn], type_ignores=[])
    ns = dict(NS)
    exec(compile(ast.fix_missing_locations(mod), REF, 'exec'), ns)
    return ns[name]


displace_positions = lift('MCDisplacementMove', 'displace_positions')
quaternion = lift('MCRotationMove', '_generate_uniform_quaternion')
rotation = lift('MCRotationMove', '_rotation_matrix_from_quaternion')
rotate_positions_fn = lift('MCRotationMove', 'rotate_positions')
apply_fn = lift('MetropolizedMove', 'apply')


class _Rot:
    @staticmethod
    def generate_random_rotation_matrix():
        return rotation(quaternion())


def rotate_positions(x):
    return rotate_positions_fn(_Rot, x)


# ---- MetropolizedMove.apply on stand-ins
class _Timer:
    def start(self, *a): pass
    def stop(self, *a): pass


class _Cache:
    def get_context(self, ts):
        return object(), None


class _Sampler:
    def __init__(self, x):
        self.positions = u.Quantity(np.array(x, np.float64), u.nanometer)

    def apply_to_context(self, context, ignore_velocities=False):
        pass


class _Thermo:
    def __init__(self, energies):
        self.energies = list(energies)

    def reduced_potential(self, context):
        return self.energies.pop(0)


class _Move:
    def __init__(self, shift):
        self.atom_subset, self.n_accepted, self.n_proposed, self.shift = [1, 2], 0, 0, shift

    def _get_context_cache(self, c):
        return _Cache()

    def _propose_positions(self, x):
        return x + u.Quantity(self.shift, u.nanometer)


NS_APPLY = apply_fn.__globals__
NS_APPLY['Timer'] = _Timer

rng = np.random.default_rng(2024)
P = rng.normal(0.0, 0.3, (5, 3)) + np.array([1.0, 2.0, 3.0])
sig = np.array([0.05, 0.5, 2.0])
randn = rng.normal(size=(3, 3))
disp = []
for s, r in zip(sig, randn):
    DRAWS.queue.append(r)
    disp.append(np.asarray(displace_positions(u.Quantity(P, u.nanometer), s * u.nanometer) / u.nanometer))
rand_q = np.vstack([rng.random((6, 3)), [[0.0, 0.25, 0.5], [1.0, 0.0, 0.75]]])
quats = []
for r in rand_q:
    DRAWS.queue.append(r)
    quats.append(quaternion())
q_cases = np.vstack([np.array(quats), rng.normal(size=(3, 4)), np.zeros((1, 4))])
mats = np.array([np.asarray(rotation(q)) for q in q_cases])
rot = []
for r in rand_q:
    DRAWS.queue.append(r)
    rot.append(np.asarray(rotate_positions(u.Quantity(P, u.nanometer)) / u.nanometer))
# accept rule: (initial reduced energy, proposed reduced energy, uniform) -> accepted?
acc_cases = np.array([[0.0, -1.0, 0.99], [0.0, 0.0, 0.99], [0.0, 1.0, 0.30], [0.0, 1.0, 0.40], [5.0, 7.5, 0.05],
                      [5.0, 7.5, 0.1], [0.0, np.nan, 0.0], [0.0, np.inf, 0.0], [0.0, 40.0, 1e-20]])
acc = []
for e0, e1, ur in acc_cases:
    mv, ss = _Move(np.array([0.1, 0.0, 0.0])), _Sampler(P)
    DRAWS.queue[:] = [[ur]]     # (a decision by dU <= 0 draws nothing)
    apply_fn(mv, _Thermo([e0, e1]), ss, None)
    moved = not np.allclose(np.asarray(ss.positions / u.nanometer), P)
    acc.append([mv.n_accepted, mv.n_proposed, int(moved)])

# constructor signatures and state keys
meta = {'signatures': {}, 'state_keys': {}}
for cls in ('MetropolizedMove', 'MCDisplacementMove', 'MCRotationMove', 'SequenceMove'):
    fn = [n for n in CLASSES[cls].body if isinstance(n, ast.FunctionDef) and n.name == '__init__'][0]
    a = fn.args
    names = [x.arg for x in a.args]
    defaults = [None] * (len(names) - len(a.defaults)) + [ast.unparse(d) for d in a.defaults]
    meta['signatures'][cls] = {'args': [[n, d] for n, d in zip(names, defaults) if n != 'self'],
                               'kwarg': a.kwarg.arg if a.kwarg else None}
    gs = [n for n in CLASSES[cls].body if isinstance(n, ast.FunctionDef) and n.name == '__getstate__']
    keys = set()
    for node in ast.walk(gs[0]) if gs else ():
        if isinstance(node, ast.Call) and getattr(node.func, 'id', None) == 'dict':
            keys |= {k.arg for k in node.keywords}
        if isinstance(node, ast.Subscript) and isinstance(node.slice, ast.Constant) and isinstance(node.ctx, ast.Store):
            keys.add(node.slice.value)
    meta['state_keys'][cls] = sorted(keys)
# the statistics keys MetropolizedMove.__getstate__ adds through self.statistics
meta['state_keys']['MetropolizedMove'] = sorted(set(meta['state_keys']['MetropolizedMove']) | {'n_accepted', 'n_proposed'})
for cls in ('MCDisplacementMove', 'MCRotationMove'):
    meta['state_keys'][cls] = sorted(set(meta['state_keys'][cls]) | set(meta['state_keys']['MetropolizedMove']))

dst = os.path.join(HERE, 'mc_moves_golden.npz')
np.savez(dst, positions=P, sigma=sig, randn=randn, displaced=np.array(disp), rand_q=rand_q, quaternions=np.array(quats),
         q_cases=q_cases, matrices=mats, rotated=np.array(rot), accept_cases=acc_cases, accepted=np.array(acc),
         meta=json.dumps(meta, sort_keys=True))
print('wrote', dst)
print(json.dumps(meta, indent=1))
