"""tests/mol_langevin_oracle.py fed the C oracles' forces against their own constrained Langevin steps (oracle.Molecule and
oracle.implicit.Molecule `langevin`, with the kernel's entry RATTLE first): the same trajectory over 25 steps, for every
constraint-cluster shape, flexible and rigid molecules, centre-of-mass removal on and off, vacuum and OBC."""
import numpy as np
import pytest
import mol_langevin_oracle as mlo
from helpers import KB, device_noise
from test_gpu_molecule import MOLECULES, oracle_run


def _toluene(model):
    from implicit_helpers import implicit_system, with_model
    s, x = implicit_system('toluene')
    return with_model(s, model), x


CASES = {
    'alanine-dipeptide': MOLECULES['alanine-dipeptide'],
    'alanine-dipeptide-flexible': MOLECULES['alanine-dipeptide-flexible'],
    'propane-AllBonds-shuffled': MOLECULES['propane-AllBonds-shuffled'],
    'waters': MOLECULES['waters'],
    'mixture-shuffled': MOLECULES['mixture-shuffled'],
    'toluene-obc1': lambda: _toluene('OBC1'),
    'toluene-obc2': lambda: _toluene('OBC2'),
}


@pytest.mark.parametrize('splitting', ['V R O R V', 'O V R V O', 'V R R O R R V'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_restatement_reproduces_the_c_oracle(name, splitting):
    from oracle import oracle, implicit
    system, x = CASES[name]()
    m = implicit.Molecule(system) if system.gb_radius is not None else oracle.Molecule(system)
    n, n_steps, dt, gamma, T = system.n_particles, 25, 0.001, 5.0, 400.0
    kT = KB * T
    rng = np.random.default_rng(11)
    v0 = rng.normal(size=x.shape) * np.sqrt(kT / m.mass)[:, None]
    noise = device_noise(77, 5, 1, n, n_steps * splitting.count('O'))
    xc, vc = x.copy(), v0.copy()
    Uc = oracle_run(m, xc, vc, noise, kT, dt, gamma, n_steps, splitting)
    cons = m.cons if len(m.cons) else None
    xp, vp, Up = mlo.run(x, v0, m.mass, kT, lambda y: m.energy(np.ascontiguousarray(y), forces=True), noise, dt, gamma,
                         n_steps, splitting, cons=cons, remove_cm=bool(system.remove_cm_motion))
    assert np.abs(xp - x).max() > 1e-3            # (the molecule moved)
    assert np.abs(xp - xc).max() <= 1e-12, np.abs(xp - xc).max()
    # (the two differ in the order of a few sums; the rigid waters' velocities part by up to 1.3e-12 of the largest)
    assert np.abs(vp - vc).max() <= 2e-12 * np.abs(vc).max(), np.abs(vp - vc).max()
    assert abs(Up - Uc) <= 1e-12 * max(1.0, abs(Uc))
