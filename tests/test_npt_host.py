"""Constant pressure on the host: pressure plumbing and refusals, the reduced potential with pV, the dispersion
coefficients, the oracle's Monte Carlo barostat step (its algebra, the refusal of small boxes, the ideal gas's volume law),
the shard format that carries boxes between ranks and the reporter's volumes record."""
import numpy as np
import pytest
from openmmtools_b200 import unit, states, alchemy, testsystems, _backend

KB = 8.31446261815324e-3   # kJ/mol/K
BAR = 0.0602214076         # kJ/mol/nm^3 per bar


def alchemical_fluid(N=64, dispersion=True):
    fluid = testsystems.LennardJonesFluid(nparticles=N)
    return alchemy.AbsoluteAlchemicalFactory(disable_alchemical_dispersion_correction=not dispersion).create_alchemical_system(
        fluid.system, alchemy.AlchemicalRegion(alchemical_atoms=range(4)))


def npt_protocol(asys, lambdas, pressures):
    return states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': lambdas, 'pressure': pressures}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=alchemy.AlchemicalState.from_system(asys))


def ideal_gas_oracle(N, box, rc=1.02):
    """The oracle's LJ fluid with epsilon = 0: no interactions, so the barostat samples the ideal gas."""
    from oracle import oracle
    return oracle.LJSystem(np.full(N, 0.34), np.zeros(N), np.full(N, 39.9), np.zeros(N, np.uint8), tuple(box), rc, rc - 0.34)


# ---- plumbing ----------------------------------------------------------------------------------------------------------------
def test_pressure_on_periodic_lj_states():
    fluid = testsystems.LennardJonesFluid(nparticles=64)
    s = states.ThermodynamicState(fluid.system, 300 * unit.kelvin, 20 * unit.bar)
    assert s.pressure == 20 * unit.bar
    assert s._pressure_md == pytest.approx(20 * BAR, rel=1e-15)
    s.pressure = 1.0 * unit.atmosphere
    assert s._pressure_md == pytest.approx(1.01325 * BAR, rel=1e-15)
    s.pressure = None
    assert s.pressure is None and s._pressure_md is None
    tstates = npt_protocol(alchemical_fluid(), [1.0, 0.5, 0.0], [10, 20, 40] * unit.bar)
    assert [t.pressure for t in tstates] == [10 * unit.bar, 20 * unit.bar, 40 * unit.bar]
    assert [t.lambda_sterics for t in tstates] == [1.0, 0.5, 0.0]
    assert tstates[0].is_state_compatible(tstates[2])


def test_pressure_refusals():
    for system in (testsystems.HarmonicOscillator().system, testsystems.AlanineDipeptideVacuum().system):
        with pytest.raises(states.ThermodynamicsError) as e:
            states.ThermodynamicState(system, 300 * unit.kelvin, 1 * unit.bar)
        assert e.value.code == states.ThermodynamicsError.BAROSTATED_NONPERIODIC
        s = states.ThermodynamicState(system, 300 * unit.kelvin)
        with pytest.raises(states.ThermodynamicsError):
            s.pressure = 1 * unit.bar
        assert s.pressure is None
    fluid = testsystems.LennardJonesFluid(nparticles=64)
    with pytest.raises(NotImplementedError):
        states.ThermodynamicState(fluid.system, 300 * unit.kelvin, 1 * unit.bar, surface_tension=1.0)
    with pytest.raises(TypeError):
        states.ThermodynamicState(fluid.system, 300 * unit.kelvin, 1.0)
    npt = states.ThermodynamicState(fluid.system, 300 * unit.kelvin, 1 * unit.bar)
    nvt = states.ThermodynamicState(fluid.system, 300 * unit.kelvin)
    assert not npt.is_state_compatible(nvt)
    with pytest.raises(states.ThermodynamicsError) as e:
        _backend.check_compatible([npt, nvt])
    assert e.value.code == states.ThermodynamicsError.INCOMPATIBLE_ENSEMBLE


@pytest.mark.parametrize('dispersion', [True, False])
def test_dispersion_coefficients_over_volume(dispersion):
    """c_l / V equals the long-range corrections evaluated at volume V, with and without the alchemical part."""
    asys = alchemical_fluid(dispersion=dispersion)
    lambdas = [1.0, 0.6, 0.2, 0.0]
    tstates = npt_protocol(asys, lambdas, [10.0] * 4 * unit.bar)
    p, c = _backend.pressure_tables(tstates)
    assert np.allclose(p, 10 * BAR, rtol=1e-15)
    for scale in (0.8, 1.0, 1.3):
        scaled = asys.copy()
        scaled.box_vectors = np.asarray(asys.box_vectors) * scale
        V = abs(np.linalg.det(scaled.box_vectors))
        for l, lam in enumerate(lambdas):
            ref = _backend.lj_dispersion_correction(scaled) + _backend.alchemical_dispersion_correction(scaled, lam)
            assert c[l] / V == pytest.approx(ref, rel=1e-12, abs=1e-14)
    assert _backend.pressure_tables(states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': lambdas}, constants={'temperature': 300.0 * unit.kelvin},
        composable_states=alchemy.AlchemicalState.from_system(asys))) is None


def test_barostat_ideal_gas_volume_law():
    """The oracle's barostat step with no interactions: the stationary volume is Gamma(N + 1, kT / p), as
    p(V) ~ V^N exp(-beta p V)."""
    from oracle import npt
    rng = np.random.default_rng(7)
    N, kT, p = 32, KB * 300.0, 40 * BAR
    Vm = (N + 1) * kT / p
    chains, n_att, burn = 32, 3000, 500
    osys = ideal_gas_oracle(N, [Vm ** (1 / 3)] * 3)
    x0 = rng.random((N, 3))
    samples = []
    for _ in range(chains):
        box = np.full(3, Vm ** (1 / 3) * 1.2)
        x = x0 * box
        st = npt.barostat_state(0.01 * np.prod(box))
        vs = []
        for a in range(n_att):
            npt.barostat_step(osys, x, box, st, rng.random(), rng.random(), 1.0, kT, p, 0.0, 0.0)
            if a >= burn:
                vs.append(np.prod(box))
        samples.append(vs)
    v = np.array(samples)
    means, variances = v.mean(axis=1), v.var(axis=1)
    se_m, se_v = means.std(ddof=1) / np.sqrt(chains), variances.std(ddof=1) / np.sqrt(chains)
    assert abs(means.mean() - Vm) < 4 * se_m, (means.mean(), Vm, se_m)
    assert abs(variances.mean() - (N + 1) * (kT / p) ** 2) < 4 * se_v


def test_barostat_step_algebra_and_refusal():
    """w = dU + c (1/V' - 1/V) + p dV - N kT ln(V'/V) on an interacting fluid; edges below min_edge are refused."""
    from oracle import npt, oracle
    from helpers import lj_setup
    s = lj_setup(N=64, n_alch=4, seed=3)
    osys = oracle.LJSystem(s['sigma'], s['eps'], s['mass'], s['alch'], tuple(s['box']), s['rc'], s['rs'])
    x, box = s['x'].copy(), s['box'].copy()
    kT, p, c = KB * 300.0, 30 * BAR, -20.0
    V = np.prod(box)
    st = npt.barostat_state(0.05 * V)
    u1 = 0.2
    r, w = npt.barostat_step(osys, x, box, st, u1, 0.999999, 0.7, kT, p, c, 0.0)
    dV = 0.05 * V * (2 * u1 - 1)
    sc = np.cbrt((V + dV) / V)
    U0 = osys.energy(s['x'], 0.7)[0]
    osys1 = oracle.LJSystem(s['sigma'], s['eps'], s['mass'], s['alch'], tuple(s['box'] * sc), s['rc'], s['rs'])
    U1 = osys1.energy(s['x'] * sc, 0.7)[0]
    ref = U1 - U0 + c * (1 / (V + dV) - 1 / V) + p * dV - 64 * kT * np.log((V + dV) / V)
    assert w == pytest.approx(ref, rel=1e-12, abs=1e-9)
    assert r == (1 if ref <= 0 else 0) and st.n_attempted == 1 and st.n_accepted == r
    if r:
        assert np.allclose(box, s['box'] * sc, rtol=1e-15) and np.allclose(x, s['x'] * sc, rtol=1e-15)
    tight = np.full(3, 2.05 * s['rc'])
    st = npt.barostat_state(0.5 * np.prod(tight))
    xt = s['x'].copy()
    r, w = npt.barostat_step(osys, xt, tight, st, 0.0, 0.0, 1.0, kT, p, c, 2 * s['rc'])
    assert r == -1 and w is None and np.array_equal(tight, np.full(3, 2.05 * s['rc'])) and st.n_attempted == 1


def test_shard_format_carries_boxes_and_barostat_state():
    from openmmtools_b200._dist import _encode_shard, _decode_shard
    rng = np.random.default_rng(1)
    rec = np.array([5.1, 5.2, 5.3, 1.25, 3, 7, 4], np.float64)
    shard = [(3, rng.random((5, 3)), rng.random((5, 3)), -1.0, 2.0, rec), (4, rng.random((5, 3)), None, None, None)]
    out = _decode_shard(_encode_shard(shard))
    assert np.array_equal(out[0][5], rec) and out[1][5] is None
    assert np.array_equal(out[0][1], shard[0][1]) and np.array_equal(out[0][2], shard[0][2]) and out[0][3:5] == (-1.0, 2.0)
    with pytest.raises(RuntimeError):
        _decode_shard(_encode_shard(shard)[:-8])


def test_reporter_volumes_record(tmp_path):
    from openmmtools_b200.multistate import MultiStateReporter
    r = MultiStateReporter(str(tmp_path / 'v.store'), open_mode='w')
    r.set_dimensions(3, 3, 10)
    for it in range(3):
        r.write_volumes(np.array([100.0, 101.0, 102.0]) + it, it)
    r.write_last_iteration(2)
    r.close()
    r2 = MultiStateReporter(str(tmp_path / 'v.store'), open_mode='r')
    assert np.array_equal(r2.read_volumes(1), [101.0, 102.0, 103.0])
    assert r2.read_volumes().shape == (3, 3)
