"""Adapter from the reference's OpenMM objects to the GPU engine (the code INTEGRATION.md sections 1-2 describe).

``system_from_openmm`` reads an ``openmm.System`` -- or any object with the same methods: the tests use the recording
stand-ins that ``tests/golden/make_alchemy_golden.py`` feeds to the reference's own ``AbsoluteAlchemicalFactory`` --
that holds a zero-charge Lennard-Jones ``NonbondedForce`` (``testsystems.LennardJonesFluid``,
/root/reference/openmmtools/testsystems.py:1956-1997), optionally alchemically modified by
``AbsoluteAlchemicalFactory._alchemically_modify_NonbondedForce`` (/root/reference/openmmtools/alchemy/alchemy.py:1539-2038):

  * the original ``NonbondedForce`` keeps every particle, with the alchemical epsilons set to zero (:1903-1909);
  * two ``CustomNonbondedForce`` objects carry the soft-core sterics: alchemical x non-alchemical (interaction group
    :1915, controlled by the global ``lambda_sterics``) and alchemical x alchemical (:1919; its expression has
    ``lambda_sterics = 1`` baked in unless ``annihilate_sterics``, :1776-1777).  Per-particle parameters are (sigma,
    epsilon); the globals ``softcore_alpha/a/b/c`` are the region's soft-core constants (:1383-1388);
  * electrostatic forces exist but are identically zero for the LJ fluid and are ignored (non-zero charges are refused);
  * with two alchemical regions each region has its own pair of soft-core forces, driven by ``lambda_sterics<suffix>``
    (:1695-1777), and no force covers the pairs across the regions; the record then carries ``alchemical_regions``.

and returns the :class:`openmmtools_b200.system.System` record the engine consumes.  ``create_engine_from_openmm`` goes
on to a configured :class:`Engine`; ``B200ReplicaExchangeSampler`` is the drop-in sampler fed with reference-side
objects.  Nothing here imports OpenMM: quantities are accepted as ``openmm.unit`` / ``openmmtools_b200.unit``
quantities or plain md-unit numbers.
"""
import re
import numpy as np
from .. import unit, _backend
from ..system import System, LJ


def _md(x, attr=None):
    """A number in md units (nm, ps, dalton, kJ/mol, e) from a quantity of either unit package or a plain number."""
    if hasattr(x, 'value_in_unit_system'):
        try:
            import openmm.unit as ou         # a real OpenMM quantity
            return x.value_in_unit_system(ou.md_unit_system)
        except ImportError:
            pass
    if isinstance(x, unit.Quantity):
        return x._md()
    return x


def _name(force):
    return type(force).__name__


def _forces(system):
    if hasattr(system, 'getForces'):
        return list(system.getForces())
    return [system.getForce(i) for i in range(system.getNumForces())]


_SOFTCORE = ('softcore_alpha', 'softcore_a', 'softcore_b', 'softcore_c')


def _globals(force):
    """{name: default} of a Custom*Force, from OpenMM's getters or from a recording stand-in."""
    if hasattr(force, 'getNumGlobalParameters'):
        return {force.getGlobalParameterName(k): force.getGlobalParameterDefaultValue(k)
                for k in range(force.getNumGlobalParameters())}
    return dict(getattr(force, 'globals', {}))


def _interaction_groups(force):
    if hasattr(force, 'getNumInteractionGroups'):
        return [tuple(sorted(s) for s in force.getInteractionGroupParameters(k)) for k in range(force.getNumInteractionGroups())]
    return [(sorted(a), sorted(b)) for a, b in getattr(force, 'groups', [])]


def _particle_parameters(force, i):
    if hasattr(force, 'getParticleParameters'):
        return list(force.getParticleParameters(i))
    return list(force.particles[i])


def _expression(force):
    return force.getEnergyFunction() if hasattr(force, 'getEnergyFunction') else force.expression


def system_from_openmm(system, forces=None):
    """The engine's parameter record for an OpenMM LJ system, plain or alchemically modified (see module docstring).

    ``forces``: the forces to read when they are not (yet) attached to ``system`` -- e.g. the dict/list that
    ``_alchemically_modify_NonbondedForce`` returns."""
    if forces is None:
        forces = _forces(system)
    elif isinstance(forces, dict):
        forces = [f for v in forces.values() for f in v]
    nb = [f for f in forces if _name(f) == 'NonbondedForce']
    if len(nb) != 1:
        raise NotImplementedError('exactly one NonbondedForce is expected (found %d)' % len(nb))
    nb = nb[0]
    n = nb.getNumParticles()
    q = np.array([_md(nb.getParticleParameters(i)[0]) for i in range(n)], dtype=np.float64)
    if np.any(q != 0.0):
        raise NotImplementedError('charged particles need an electrostatics kernel (PME / reaction field): not on this path')
    if nb.getNumExceptions() != 0:
        raise NotImplementedError('nonbonded exceptions (bonded molecules) are not on this path')
    if nb.getNonbondedMethod() != type(nb).CutoffPeriodic:
        raise NotImplementedError('only NonbondedForce.CutoffPeriodic is provided')
    sigma = np.array([_md(nb.getParticleParameters(i)[1]) for i in range(n)], dtype=np.float64)
    eps = np.array([_md(nb.getParticleParameters(i)[2]) for i in range(n)], dtype=np.float64)
    masses = [_md(system.getParticleMass(i)) for i in range(n)]
    box = np.array([[_md(c) for c in _md(v)] for v in system.getDefaultPeriodicBoxVectors()], dtype=np.float64)
    out = System(LJ, masses, box)
    out.charge = q
    out.cutoff = float(_md(nb.getCutoffDistance()))
    out.use_switching_function = bool(nb.getUseSwitchingFunction())
    out.switching_distance = float(_md(nb.getSwitchingDistance())) if out.use_switching_function else out.cutoff
    out.use_dispersion_correction = bool(nb.getUseDispersionCorrection())

    # ---- alchemical sterics: the CustomNonbondedForces whose expression is the soft-core Lennard-Jones of alchemy.py:1379-1388
    steric = []
    for f in forces:
        if _name(f) != 'CustomNonbondedForce':
            continue
        g = _globals(f)
        if all(k in g for k in _SOFTCORE) and 'reff_sterics' in _expression(f):
            steric.append(f)
        elif len(getattr(f, 'particles', [])) or (hasattr(f, 'getNumParticles') and f.getNumParticles()):
            # electrostatic CustomNonbondedForces of the factory: every charge product must vanish
            pass
    for f in forces:
        if _name(f) == 'CustomBondForce' and (len(getattr(f, 'bonds', [])) or (hasattr(f, 'getNumBonds') and f.getNumBonds())):
            raise NotImplementedError('alchemical exceptions (CustomBondForce with bonds) are not on this path')
    if not steric:
        out.sigma, out.epsilon = sigma, eps
        return out
    # One environment x region force and one region x region force per region (alchemy.py:1752-1777, 1915-1919), in the
    # order of the regions; a region's lambda is the global lambda_sterics<suffix> of its environment x region force.
    regions, soft = [], None      # regions: [atoms, lambda name or None, annihilate]
    def region_of(atoms):
        for r in regions:
            if r[0] == atoms:
                return r
        if any(r[0] & atoms for r in regions):
            raise NotImplementedError('the soft-core forces disagree on the alchemical atoms')
        regions.append([atoms, None, None])
        return regions[-1]
    lambdas = lambda g: [k for k in g if re.fullmatch(r'lambda_sterics(_.+)?', k)]
    for f in steric:
        groups = _interaction_groups(f)
        if len(groups) != 1:
            raise NotImplementedError('one interaction group per soft-core force is expected')
        a, b = (set(groups[0][0]), set(groups[0][1]))
        g = _globals(f)
        sc = tuple(float(_md(g[k])) for k in _SOFTCORE)
        if soft is not None and sc != soft:
            raise NotImplementedError('the soft-core forces disagree on the soft-core constants')
        soft = sc
        if a == b:          # region x region (alchemy.py:1919): lambda is a free global only when annihilating
            r = region_of(a)
            names = lambdas(g)
            r[2] = bool(names) and not re.search(re.escape(names[0]) + r'\s*=\s*1(\.0*)?\s*;', _expression(f))
        else:               # region x environment (alchemy.py:1915)
            if a & b:
                raise NotImplementedError('overlapping interaction groups')
            r = region_of(a if len(a) <= len(b) else b)
            names = lambdas(g)
            if len(names) != 1:
                raise NotImplementedError('an environment x region soft-core force needs one lambda_sterics parameter')
            r[1] = names[0]
        # the original sigma / epsilon of the alchemical atoms live in the custom force (zeroed in the NonbondedForce)
        for i in sorted(r[0]):
            p = _particle_parameters(f, i)
            sigma[i], eps[i] = float(_md(p[0])), float(_md(p[1]))
    if len(regions) > 2:
        raise NotImplementedError('more than two alchemical regions are not provided')
    names = [r[1] or 'lambda_sterics' for r in regions]
    if len(set(names)) != len(names):
        raise NotImplementedError('two alchemical regions with the same lambda_sterics parameter')
    out.sigma, out.epsilon = sigma, eps
    out.alchemical_atoms = tuple(sorted(int(i) for r in regions for i in r[0]))
    out.annihilate_sterics = bool(regions[0][2])
    out.softcore_alpha, out.softcore_a, out.softcore_b, out.softcore_c = soft
    lrc = [bool(f.getUseLongRangeCorrection()) if hasattr(f, 'getUseLongRangeCorrection') else bool(getattr(f, 'lrc', False)) for f in steric]
    out.alchemical_dispersion_correction = any(lrc)
    if len(regions) == 1:
        out.global_parameters = {'lambda_sterics': 1.0, 'lambda_electrostatics': 1.0}
        return out
    out.alchemical_regions = tuple((None if n == 'lambda_sterics' else n[len('lambda_sterics_'):],
                                    tuple(sorted(int(i) for i in r[0])), bool(r[2])) for n, r in zip(names, regions))
    out.global_parameters = {}
    for n in names:
        out.global_parameters[n] = 1.0
        out.global_parameters[n.replace('sterics', 'electrostatics')] = 1.0
    return out


def thermodynamic_states_from_openmm(system_record, temperatures, lambda_sterics=None, lambda_sterics_2=None):
    """Our ThermodynamicState objects (one per state) for the record: temperatures in kelvin (numbers or quantities), and
    for an alchemical record the lambda_sterics of every state (with two regions: of the first region, and
    ``lambda_sterics_2`` of the second)."""
    from .. import states, alchemy
    temps = [float(_md(t)) for t in temperatures]
    if system_record.alchemical_regions is not None:
        if lambda_sterics is None or lambda_sterics_2 is None or not (len(lambda_sterics) == len(lambda_sterics_2) == len(temps)):
            raise ValueError('one lambda_sterics and one lambda_sterics_2 per state are needed for two alchemical regions')
        out = []
        for T, lams in zip(temps, zip(lambda_sterics, lambda_sterics_2)):
            comp = []
            for (name, _, _), lam in zip(system_record.alchemical_regions, lams):
                a = alchemy.AlchemicalState.from_system(system_record, parameters_name_suffix=name)
                sfx = '' if name is None else '_' + name
                setattr(a, 'lambda_sterics' + sfx, float(lam))
                setattr(a, 'lambda_electrostatics' + sfx, float(lam))
                comp.append(a)
            out.append(states.CompoundThermodynamicState(states.ThermodynamicState(system_record, T * unit.kelvin), comp))
        return out
    if lambda_sterics_2 is not None:
        raise ValueError('lambda_sterics_2 needs a system with two alchemical regions')
    if system_record.is_alchemical:
        if lambda_sterics is None or len(lambda_sterics) != len(temps):
            raise ValueError('one lambda_sterics per state is needed for an alchemical system')
        out = []
        for T, lam in zip(temps, lambda_sterics):
            a = alchemy.AlchemicalState.from_system(system_record)
            a.lambda_sterics = float(lam)
            a.lambda_electrostatics = float(lam)
            out.append(states.CompoundThermodynamicState(states.ThermodynamicState(system_record, T * unit.kelvin), [a]))
        return out
    return [states.ThermodynamicState(system_record, T * unit.kelvin) for T in temps]


def create_engine_from_openmm(system, temperatures, lambda_sterics=None, n_replicas=None, forces=None, device=0,
                              rank=0, world_size=1, lambda_sterics_2=None):
    """``rx_create`` + ``rx_set_particles`` + ``rx_set_states`` from OpenMM objects (INTEGRATION.md section 2): returns
    ``(engine, system_record, thermodynamic_states)``; positions, integrator and the mixing seed are the caller's.
    Two alchemical regions take the second region's lambdas as ``lambda_sterics_2``."""
    rec = system_from_openmm(system, forces)
    tstates = thermodynamic_states_from_openmm(rec, temperatures, lambda_sterics, lambda_sterics_2)
    eng = _backend.build_engine(tstates, n_replicas or len(tstates), device=device, rank=rank, world_size=world_size)
    return eng, rec, tstates


def B200ReplicaExchangeSampler(openmm_thermodynamic_states, openmm_sampler_states, mcmc_move, **sampler_kwargs):
    """The drop-in: reference-side ``ThermodynamicState`` / ``SamplerState`` / ``LangevinSplittingDynamicsMove`` objects
    (openmmtools over OpenMM) in, a created :class:`openmmtools_b200.multistate.ReplicaExchangeSampler` out.  The
    lambdas are read from the compound states' ``lambda_sterics``, temperatures from ``.temperature``, positions /
    velocities / box vectors from the sampler states, the integrator parameters from the move."""
    from .. import states, mcmc, multistate
    ts = list(openmm_thermodynamic_states)
    rec = system_from_openmm(ts[0].get_system(remove_thermostat=True) if hasattr(ts[0], 'get_system') else ts[0].system)
    temps = [t.temperature for t in ts]
    lams = [getattr(t, 'lambda_sterics', 1.0) for t in ts] if rec.is_alchemical else None
    tstates = thermodynamic_states_from_openmm(rec, temps, lams)
    sstates = []
    for s in ([openmm_sampler_states] if not isinstance(openmm_sampler_states, (list, tuple)) else openmm_sampler_states):
        bv = s.box_vectors
        sstates.append(states.SamplerState(np.asarray(_md(s.positions), dtype=np.float64) * unit.nanometer,
                                           velocities=None if s.velocities is None else np.asarray(_md(s.velocities), dtype=np.float64) * (unit.nanometer / unit.picosecond),
                                           box_vectors=None if bv is None else np.asarray(_md(bv), dtype=np.float64) * unit.nanometer))
    move = mcmc.LangevinSplittingDynamicsMove(timestep=float(_md(mcmc_move.timestep)) * unit.picosecond,
                                              collision_rate=float(_md(mcmc_move.collision_rate)) / unit.picosecond,
                                              n_steps=int(mcmc_move.n_steps), reassign_velocities=bool(mcmc_move.reassign_velocities),
                                              splitting=getattr(mcmc_move, 'splitting', 'V R O R V'))
    sampler = multistate.ReplicaExchangeSampler(mcmc_moves=move, **sampler_kwargs)
    sampler.create(tstates, sstates)
    return sampler
