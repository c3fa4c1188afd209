"""The anisotropic Monte Carlo barostat on the host: the MonteCarloAnisotropicBarostat / MonteCarloBarostat records, the
refusals ThermodynamicState raises for them, compatibility and protocols, the engine calls build_engine makes for each
barostat, and the oracle's anisotropic step (its algebra, the refusal of a short scaled edge, the z-only ideal gas)."""
import copy
import pickle
import numpy as np
import pytest
from openmmtools_b200 import unit, states, alchemy, testsystems, _backend
from openmmtools_b200.system import MonteCarloBarostat, MonteCarloAnisotropicBarostat
from test_npt_host import KB, BAR, alchemical_fluid, ideal_gas_oracle

TE = states.ThermodynamicsError


def fluid_with(*barostats, N=64):
    system = testsystems.LennardJonesFluid(nparticles=N).system
    for b in barostats:
        system.addForce(b)
    return system


def aniso(p=20.0, scale=(True, True, True), frequency=25):
    return MonteCarloAnisotropicBarostat(p * unit.bar if np.isscalar(p) else [q * unit.bar for q in p], 300 * unit.kelvin,
                                         *scale, frequency=frequency)


# ---- records and refusals ----------------------------------------------------------------------------------------------------
def test_anisotropic_record_getters_and_setters():
    b = MonteCarloAnisotropicBarostat([1.0, 2.0, 3.0] * unit.bar, 310 * unit.kelvin, True, False, True, 25)
    assert np.array_equal(b.getDefaultPressure().value_in_unit(unit.bar), [1.0, 2.0, 3.0])
    assert (b.getScaleX(), b.getScaleY(), b.getScaleZ()) == (True, False, True) and b.getFrequency() == 25
    assert b.getDefaultTemperature() == 310 * unit.kelvin
    b.setDefaultPressure(5 * unit.bar)
    assert np.array_equal(b.getDefaultPressure().value_in_unit(unit.bar), [5.0, 5.0, 5.0])
    b.setScaleY(True)
    b.setFrequency(50)
    assert b.getScaleY() and b.getFrequency() == 50
    with pytest.raises(TypeError):
        b.setDefaultPressure(1.0)
    i = MonteCarloBarostat(2 * unit.bar, 300 * unit.kelvin)
    assert i.getDefaultPressure() == 2 * unit.bar and i.getFrequency() == 25
    system = fluid_with()
    assert system.addForce(b) == 0 and system.getNumForces() == 1 and system.getForces()[0] is b
    system.removeForce(0)
    assert system.getForces() == []
    with pytest.raises(NotImplementedError):
        system.addForce(object())


def test_anisotropic_state_pressure_from_the_record():
    s = states.ThermodynamicState(fluid_with(aniso([7.0, 9.0, 7.0], (True, False, True))), 300 * unit.kelvin)
    assert s.pressure == 7 * unit.bar and s._barostat_scale == (True, False, True)
    assert s.barostat.getScaleY() is False
    s.pressure = 12 * unit.bar          # all three axes
    assert np.array_equal(s.barostat.getDefaultPressure().value_in_unit(unit.bar), [12.0] * 3)
    rec = s.system.getForces()
    assert len(rec) == 1 and np.array_equal(rec[0].getDefaultPressure().value_in_unit(unit.bar), [12.0] * 3)
    assert (rec[0].getScaleX(), rec[0].getScaleY(), rec[0].getScaleZ()) == (True, False, True)
    assert states.ThermodynamicState(s.system, 300 * unit.kelvin).is_state_compatible(s)
    # the pressure argument wins over the record's
    assert states.ThermodynamicState(fluid_with(aniso(7.0)), 300 * unit.kelvin, 3 * unit.bar).pressure == 3 * unit.bar
    s.pressure = None                   # removes the barostat: an NVT state like one without a record
    nvt = states.ThermodynamicState(fluid_with(), 300 * unit.kelvin)
    assert s.pressure is None and s.barostat is None and s.system.getForces() == []
    assert s.is_state_compatible(nvt) and s._standard_system_hash == nvt._standard_system_hash


def test_refusals():
    for bad in (aniso(20.0, (False, False, False)), aniso([10.0, 11.0, 10.0])):
        with pytest.raises(TE) as e:
            states.ThermodynamicState(fluid_with(bad), 300 * unit.kelvin)
        assert e.value.code == TE.UNSUPPORTED_ANISOTROPIC_BAROSTAT
    # the unscaled axis's pressure is ignored
    assert states.ThermodynamicState(fluid_with(aniso([10.0, 99.0, 10.0], (True, False, True))),
                                     300 * unit.kelvin).pressure == 10 * unit.bar
    for b in (aniso(frequency=50), MonteCarloBarostat(1 * unit.bar, 300 * unit.kelvin, 10)):
        with pytest.raises(NotImplementedError):
            states.ThermodynamicState(fluid_with(b), 300 * unit.kelvin)
    for system in (testsystems.HarmonicOscillator().system, testsystems.AlanineDipeptideVacuum().system):
        for b in (aniso(), MonteCarloBarostat(1 * unit.bar, 300 * unit.kelvin)):
            system = system.copy()
            system.forces = []
            system.addForce(b)
            with pytest.raises(TE) as e:
                states.ThermodynamicState(system, 300 * unit.kelvin)
            assert e.value.code == TE.BAROSTATED_NONPERIODIC
    with pytest.raises(TE) as e:
        states.ThermodynamicState(fluid_with(aniso(), MonteCarloBarostat(1 * unit.bar, 300 * unit.kelvin)), 300 * unit.kelvin)
    assert e.value.code == TE.MULTIPLE_BAROSTATS


def test_compatibility():
    T = 300 * unit.kelvin
    iso = states.ThermodynamicState(fluid_with(), T, 20 * unit.bar)
    iso_rec = states.ThermodynamicState(fluid_with(MonteCarloBarostat(30 * unit.bar, T)), T)
    xyz, xyz2 = (states.ThermodynamicState(fluid_with(aniso(p)), T) for p in (20.0, 45.0))
    z = states.ThermodynamicState(fluid_with(aniso(20.0, (False, False, True))), T)
    assert iso.is_state_compatible(iso_rec)
    assert not iso.is_state_compatible(xyz) and not xyz.is_state_compatible(iso)
    assert xyz.is_state_compatible(xyz2)            # pressures differ only
    assert not xyz.is_state_compatible(z)
    for pair in ([iso, xyz], [xyz, z]):
        with pytest.raises(TE) as e:
            _backend.check_compatible(pair)
        assert e.value.code == TE.INCOMPATIBLE_ENSEMBLE
    system = fluid_with(aniso())
    h = system.standard_hash()
    system.getForce(0).setDefaultPressure(99 * unit.bar)
    assert system.standard_hash() == h
    system.getForce(0).setScaleX(False)
    assert system.standard_hash() != h
    assert fluid_with().standard_hash() == testsystems.LennardJonesFluid(nparticles=64).system.standard_hash()


def test_protocol_keeps_the_scaled_axes_and_pickles():
    asys = alchemical_fluid()
    asys.addForce(aniso(20.0, (False, False, True)))
    tstates = states.create_thermodynamic_state_protocol(
        asys, {'lambda_sterics': [1.0, 0.5, 0.0], 'pressure': [10, 20, 40] * unit.bar},
        constants={'temperature': 300.0 * unit.kelvin}, composable_states=alchemy.AlchemicalState.from_system(asys))
    assert [t.pressure for t in tstates] == [10 * unit.bar, 20 * unit.bar, 40 * unit.bar]
    assert all(t._barostat_scale == (False, False, True) for t in tstates)
    assert tstates[0].is_state_compatible(tstates[2])
    for t in tstates:
        for u in (pickle.loads(pickle.dumps(t)), copy.deepcopy(t)):
            assert u._barostat_scale == t._barostat_scale and u.pressure == t.pressure
            assert u.is_state_compatible(t) and u.lambda_sterics == t.lambda_sterics
    system = pickle.loads(pickle.dumps(asys))
    b = system.getForces()[0]
    assert isinstance(b, MonteCarloAnisotropicBarostat) and (b.getScaleX(), b.getScaleZ()) == (False, True)
    assert system.standard_hash() == asys.standard_hash() and asys.copy().standard_hash() == asys.standard_hash()


# ---- the engine calls of each barostat ---------------------------------------------------------------------------------------
class RecordingEngine:
    """Stands in for _engine.Engine: records every call build_engine makes."""
    log = []

    def __init__(self, *args, **kw):
        RecordingEngine.log.append(('__init__', args, kw))

    def __getattr__(self, name):
        return lambda *a, **k: RecordingEngine.log.append((name, a, k))


def engine_calls(monkeypatch, tstates):
    monkeypatch.setattr(_backend, 'Engine', RecordingEngine)
    RecordingEngine.log = []
    _backend.build_engine(tstates, len(tstates))
    return RecordingEngine.log


def same_calls(a, b):
    def norm(v):
        if isinstance(v, dict):
            return {k: norm(x) for k, x in v.items()}
        if isinstance(v, (list, tuple)):
            return [norm(x) for x in v]
        return np.asarray(v).tolist() if isinstance(v, np.ndarray) else v
    return norm(a) == norm(b)


def test_engine_calls_of_each_barostat(monkeypatch):
    def protocol(system, pressures):
        return states.create_thermodynamic_state_protocol(
            system, {'lambda_sterics': [1.0, 0.5, 0.0], 'pressure': pressures}, constants={'temperature': 300.0 * unit.kelvin},
            composable_states=alchemy.AlchemicalState.from_system(system))
    p = [10, 20, 40] * unit.bar
    plain = alchemical_fluid()
    ref = engine_calls(monkeypatch, protocol(plain, p))
    assert [c[0] for c in ref][-2:] == ['set_states', 'set_pressures']
    iso = alchemical_fluid()
    iso.addForce(MonteCarloBarostat(99 * unit.bar, 300 * unit.kelvin))
    assert same_calls(engine_calls(monkeypatch, protocol(iso, p)), ref)
    # a record's own pressure: the same tables as the pressure argument
    one = states.ThermodynamicState(iso, 300 * unit.kelvin)
    assert same_calls(engine_calls(monkeypatch, [one]),
                      engine_calls(monkeypatch, [states.ThermodynamicState(plain, 300 * unit.kelvin, 99 * unit.bar)]))
    for scale in ((True, True, True), (False, False, True), (True, True, False)):
        an = alchemical_fluid()
        an.addForce(aniso(5.0, scale))
        calls = engine_calls(monkeypatch, protocol(an, p))
        assert same_calls(calls[:-1], ref) and same_calls(calls[-1], ('set_anisotropic_barostat', (scale,), {}))


# ---- the oracle's anisotropic step -------------------------------------------------------------------------------------------
def test_aniso_step_algebra_and_refusal():
    """w of a one-axis proposal on an interacting fluid; only that coordinate and edge change; a short scaled edge is
    refused while an unscaled edge below the limit is not looked at."""
    from oracle import npt_aniso, oracle
    from helpers import lj_setup
    s = lj_setup(N=64, n_alch=4, seed=3)
    kT, p, c = KB * 300.0, 30 * BAR, -20.0
    V = np.prod(s['box'])
    for axis in range(3):
        osys = oracle.LJSystem(s['sigma'], s['eps'], s['mass'], s['alch'], tuple(s['box']), s['rc'], s['rs'])
        x, box = s['x'].copy(), s['box'].copy()
        st = npt_aniso.barostat_state([0.01 * V, 0.05 * V, 0.03 * V])
        u1 = 0.2
        r, w = npt_aniso.barostat_step(osys, x, box, st, axis, u1, 1e-300, 0.7, kT, p, c, 0.0)
        dV = st.volume_scale[axis] * (2 * u1 - 1)
        f = np.ones(3)
        f[axis] = (V + dV) / V
        osys1 = oracle.LJSystem(s['sigma'], s['eps'], s['mass'], s['alch'], tuple(s['box'] * f), s['rc'], s['rs'])
        ref = (osys1.energy(s['x'] * f, 0.7)[0] - osys.energy(s['x'], 0.7)[0] + c * (1 / (V + dV) - 1 / V) + p * dV
               - 64 * kT * np.log((V + dV) / V))
        assert w == pytest.approx(ref, rel=1e-12, abs=1e-9) and r == 1
        assert np.array_equal(box, s['box'] * f) and np.array_equal(x, s['x'] * f)
        assert list(st.n_attempted) == [int(a == axis) for a in range(3)] and list(st.n_accepted) == list(st.n_attempted)
    osys = oracle.LJSystem(s['sigma'], s['eps'], s['mass'], s['alch'], tuple(s['box']), s['rc'], s['rs'])
    tight = np.array([1.5 * s['rc'], 2.05 * s['rc'], 3.0 * s['rc']])
    st = npt_aniso.barostat_state(0.5 * np.prod(tight))
    r, w = npt_aniso.barostat_step(osys, s['x'].copy(), tight, st, 1, 0.0, 0.0, 1.0, kT, p, c, 2 * s['rc'])
    assert r == -1 and w is None and st.n_attempted[1] == 1
    r, w = npt_aniso.barostat_step(osys, s['x'].copy(), tight, st, 2, 0.4, 0.0, 1.0, kT, p, c, 2 * s['rc'])
    assert r in (0, 1) and w is not None      # the x edge is below the limit but not scaled


def test_aniso_adaptation_per_axis():
    """Each axis adapts at its own 10th attempt: all rejected -> / 1.1, all accepted -> * 1.1 capped at 0.3 V."""
    from oracle import npt_aniso
    N, kT = 16, KB * 300.0
    box0 = np.array([6.0, 6.0, 6.0])
    osys = ideal_gas_oracle(N, box0)
    V = np.prod(box0)
    st = npt_aniso.barostat_state([0.01 * V, 0.29 * V, 0.01 * V])
    x = np.random.default_rng(0).random((N, 3)) * box0
    box = box0.copy()
    for i in range(10):        # axis 0: proposals that are never accepted (u2 = 1 and w > 0 from a huge pressure)
        npt_aniso.barostat_step(osys, x, box, st, 0, 0.9999, 1.0, 1.0, kT, 1e6, 0.0, 0.0)
    assert st.volume_scale[0] == pytest.approx(0.01 * V / 1.1, rel=1e-15) and st.n_attempted[0] == 0
    for i in range(10):        # axis 1: always accepted (u1 = 0.5 - tiny: dV ~ 0, w ~ 0 -> accepted), capped at 0.3 V
        npt_aniso.barostat_step(osys, x, box, st, 1, 0.5, 0.0, 1.0, kT, 1e-9, 0.0, 0.0)
    assert st.volume_scale[1] == pytest.approx(0.3 * np.prod(box), rel=1e-9) and st.n_attempted[1] == 0
    assert st.volume_scale[2] == 0.01 * V and st.n_attempted[2] == 0


def test_z_only_ideal_gas_volume_law():
    """The oracle's z-only barostat with no interactions: V ~ Gamma(N + 1, kT / p), and x and y edges never change."""
    from oracle import npt_aniso
    rng = np.random.default_rng(11)
    N, kT, p = 32, KB * 300.0, 40 * BAR
    Vm = (N + 1) * kT / p
    chains, n_att, burn = 32, 3000, 500
    L = Vm ** (1 / 3)
    osys = ideal_gas_oracle(N, [L] * 3)
    x0 = rng.random((N, 3))
    samples = []
    for _ in range(chains):
        box = np.array([L, L, 1.3 * L])
        x = x0 * box
        xy = x[:, :2].copy()
        st = npt_aniso.barostat_state(0.01 * np.prod(box), scale_mask=4)
        vs = []
        for a in range(n_att):
            npt_aniso.barostat_step(osys, x, box, st, 2, rng.random(), rng.random(), 1.0, kT, p, 0.0, 0.0)
            if a >= burn:
                vs.append(np.prod(box))
        assert box[0] == L and box[1] == L and np.array_equal(x[:, :2], xy)
        samples.append(vs)
    v = np.array(samples)
    means, variances = v.mean(axis=1), v.var(axis=1)
    se_m, se_v = means.std(ddof=1) / np.sqrt(chains), variances.std(ddof=1) / np.sqrt(chains)
    assert abs(means.mean() - Vm) < 4 * se_m, (means.mean(), Vm, se_m)
    assert abs(variances.mean() - (N + 1) * (kT / p) ** 2) < 4 * se_v
