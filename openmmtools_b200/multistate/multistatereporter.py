"""MultiStateReporter: analysis + checkpoint storage for the multistate samplers, without netCDF4.

Mirrors the part of /root/reference/openmmtools/multistate/multistatereporter.py the samplers use
(``write_energies`` :865, ``write_replica_thermodynamic_states`` :763, ``write_mixing_statistics`` :957,
``write_sampler_states`` :664, ``write_last_iteration`` :1184, ``read_*`` counterparts, ``read_checkpoint_iterations``,
``write_dict``/``read_dict``, ``write_thermodynamic_states``, ``write_mcmc_moves``, ``checkpoint_interval`` :131) with
the reference's variable names and dtypes (``energies`` f8[iteration, replica, state], ``neighborhoods`` i1,
``states`` i4[iteration, replica], ``accepted``/``proposed`` i4[iteration, state, state], ``last_iteration``).

netCDF4 is not a dependency (it is not installable in the build environment), so the container is a directory:

    <storage>/meta.json                   shapes, options, metadata
    <storage>/analysis/<name>.bin         fixed-size records appended per iteration (numpy ``fromfile`` readable)
    <storage>/analysis/last_iteration     commit marker, written last (reference: between two syncs, :1199-1201)
    <storage>/checkpoint/ckpt_<it>.npz    positions, velocities, box vectors (+ RNG positions: the reference stores no
                                          RNG state, so its resumed runs are not reproducible; ours are)
    <storage>/objects.pkl                 pickled thermodynamic states and MCMC moves

Only rank 0 writes (as in the reference, multistatesampler.py:1169-1187).
"""
import json
import os
import re
import shutil
import pickle
import numpy as np
from .. import states as _states
from .. import unit


class MultiStateReporter:
    _VARS = {  # name -> (dtype, shape builder from (K, M))
        'energies': ('f8', lambda K, M: (K, M)),
        'neighborhoods': ('i1', lambda K, M: (K, M)),
        'states': ('i4', lambda K, M: (K,)),
        'accepted': ('i4', lambda K, M: (M, M)),
        'proposed': ('i4', lambda K, M: (M, M)),
        'volumes': ('f8', lambda K, M: (K,)),      # constant-pressure runs only
    }

    def __init__(self, storage, open_mode=None, checkpoint_interval=50, checkpoint_storage=None,
                 analysis_particle_indices=(), position_interval=1, velocity_interval=1):
        self._storage = str(storage)
        self._checkpoint_interval = int(checkpoint_interval)
        self._analysis_particle_indices = tuple(int(i) for i in analysis_particle_indices)
        self._position_interval = int(position_interval)    # multistatereporter.py:109-116: 0 disables the stream
        self._velocity_interval = int(velocity_interval)
        self._open_mode = None
        self._meta = None
        self._dirty = set()
        self._overwrite_statistics = False
        if open_mode is not None:
            self.open(open_mode)

    # -- properties of the reference
    @property
    def filepath(self):
        return self._storage

    @property
    def checkpoint_interval(self):
        return self._checkpoint_interval

    @property
    def analysis_particle_indices(self):
        return self._analysis_particle_indices

    @property
    def position_interval(self):
        return self._position_interval

    @property
    def velocity_interval(self):
        return self._velocity_interval

    def wants_analysis_states(self, iteration):
        """True when positions or velocities of the analysis particles are due at this iteration
        (multistatereporter.py:1686-1692)."""
        if not self._analysis_particle_indices:
            return False
        it = int(iteration)
        return (self._position_interval != 0 and it % self._position_interval == 0) or \
               (self._velocity_interval != 0 and it % self._velocity_interval == 0)

    def storage_exists(self, skip_size=False):
        return os.path.exists(os.path.join(self._storage, 'meta.json'))

    def is_open(self):
        return self._open_mode is not None

    def open(self, mode='r', convention='ReplicaExchange', netcdf_format=None):
        if mode not in ('r', 'w', 'a'):
            raise ValueError("open_mode must be 'r', 'w' or 'a'")
        if mode == 'w':
            os.makedirs(os.path.join(self._storage, 'analysis'), exist_ok=True)
            os.makedirs(os.path.join(self._storage, 'checkpoint'), exist_ok=True)
            # a fresh container (MultiStateSampler.create refuses to get here when the storage exists): sub-directories
            # such as analysis/online/ are removed as a whole
            for sub in ('analysis', 'checkpoint'):
                shutil.rmtree(os.path.join(self._storage, sub))
                os.makedirs(os.path.join(self._storage, sub))
            self._meta = {'convention': convention, 'dicts': {}}
            self._write_meta()
            self._overwrite_statistics = True    # a fresh run starts a new real-time statistics file
        else:
            if not self.storage_exists():
                raise IOError('storage {} does not exist'.format(self._storage))
            self._meta = json.load(open(os.path.join(self._storage, 'meta.json')))
            if 'checkpoint_interval' in self._meta:
                self._checkpoint_interval = int(self._meta['checkpoint_interval'])
            # an existing file keeps its analysis-particle settings (the reference reads them back from the .nc file)
            if 'analysis_particle_indices' in self._meta:
                self._analysis_particle_indices = tuple(self._meta['analysis_particle_indices'])
                self._position_interval = int(self._meta.get('position_interval', 1))
                self._velocity_interval = int(self._meta.get('velocity_interval', 1))
        self._open_mode = mode

    def close(self):
        self._open_mode = None

    def sync(self):
        pass   # data files are fsync'ed by write_last_iteration, right before the commit marker

    def __del__(self):
        self.close()

    # -- helpers
    def _write_meta(self):
        self._meta['checkpoint_interval'] = self._checkpoint_interval
        self._meta['analysis_particle_indices'] = list(self._analysis_particle_indices)
        self._meta['position_interval'] = self._position_interval
        self._meta['velocity_interval'] = self._velocity_interval
        tmp = os.path.join(self._storage, 'meta.json.tmp')
        with open(tmp, 'w') as f:
            json.dump(self._meta, f)
            f.flush(); os.fsync(f.fileno())
        os.replace(tmp, os.path.join(self._storage, 'meta.json'))

    def _path(self, name):
        return os.path.join(self._storage, 'analysis', name + '.bin')

    def _shape(self, name):
        K, M = self._meta['n_replicas'], self._meta['n_states']
        return self._VARS[name][1](K, M)

    def _write_record(self, name, iteration, array):
        dtype = np.dtype(self._VARS[name][0])
        a = np.ascontiguousarray(array, dtype=dtype)
        if 'n_replicas' not in self._meta:
            raise RuntimeError('write_thermodynamic_states / set_dimensions must be called first')
        if a.shape != tuple(self._shape(name)):
            raise ValueError('{}: expected shape {}, got {}'.format(name, self._shape(name), a.shape))
        mode = 'r+b' if os.path.exists(self._path(name)) else 'w+b'
        with open(self._path(name), mode) as f:
            f.seek(int(iteration) * a.nbytes)
            f.write(a.tobytes())
        self._dirty.add(self._path(name))

    def _read_record(self, name, iteration):
        dtype = np.dtype(self._VARS[name][0])
        shape = tuple(self._shape(name))
        rec = int(np.prod(shape)) * dtype.itemsize
        n = os.path.getsize(self._path(name)) // rec
        data = np.fromfile(self._path(name), dtype=dtype, count=n * int(np.prod(shape))).reshape((n,) + shape)
        last = self.read_last_iteration(last_checkpoint=False)
        data = data[:last + 1]     # never expose records past the commit marker
        if iteration is None:
            iteration = slice(None)
        if isinstance(iteration, (int, np.integer)) and iteration < 0:
            iteration = last + 1 + iteration
        return data[iteration]

    def set_dimensions(self, n_replicas, n_states, n_particles):
        self._meta.update(n_replicas=int(n_replicas), n_states=int(n_states), n_particles=int(n_particles))
        self._write_meta()

    # -- objects
    def write_thermodynamic_states(self, thermodynamic_states, unsampled_states):
        with open(os.path.join(self._storage, 'objects_states.pkl'), 'wb') as f:
            pickle.dump((thermodynamic_states, unsampled_states), f)

    def read_thermodynamic_states(self):
        with open(os.path.join(self._storage, 'objects_states.pkl'), 'rb') as f:
            return _restricted_load(f)

    def write_mcmc_moves(self, mcmc_moves):
        with open(os.path.join(self._storage, 'objects_moves.pkl'), 'wb') as f:
            pickle.dump(mcmc_moves, f)

    def read_mcmc_moves(self):
        with open(os.path.join(self._storage, 'objects_moves.pkl'), 'rb') as f:
            return _restricted_load(f)

    def write_dict(self, name, data, fixed_dimension=False):
        self._meta['dicts'][name] = _jsonable(data)
        self._write_meta()

    def read_dict(self, name):
        return self._meta['dicts'].get(name)

    # -- per-iteration analysis data (reference variable names)
    def write_energies(self, energy_thermodynamic_states, energy_neighborhoods, energy_unsampled_states, iteration):
        self._write_record('energies', iteration, energy_thermodynamic_states)
        self._write_record('neighborhoods', iteration, energy_neighborhoods)
        eu = np.ascontiguousarray(energy_unsampled_states, dtype=np.float64)
        if eu.size:     # reference variable 'unsampled_energies' f8[iteration, replica, unsampled]
            self._meta.setdefault('n_unsampled', int(eu.shape[1]))
            if self._meta.get('_wrote_n_unsampled') is None:
                self._meta['_wrote_n_unsampled'] = True
                self._write_meta()
            with open(self._path('unsampled_energies'), 'r+b' if os.path.exists(self._path('unsampled_energies')) else 'w+b') as f:
                f.seek(int(iteration) * eu.nbytes)
                f.write(eu.tobytes())
            self._dirty.add(self._path('unsampled_energies'))

    def read_unsampled_energies(self, iteration):
        n = self._meta.get('n_unsampled', 0)
        if not n or not os.path.exists(self._path('unsampled_energies')):
            return None
        K = self._meta['n_replicas']
        data = np.fromfile(self._path('unsampled_energies'), dtype=np.float64)
        data = data[:(data.size // (K * n)) * K * n].reshape(-1, K, n)
        return data[iteration]

    def read_energies(self, iteration=slice(None)):
        e = self._read_record('energies', iteration)
        n = self._read_record('neighborhoods', iteration)
        unsampled = self.read_unsampled_energies(iteration)
        if unsampled is None:
            unsampled = np.zeros(e.shape[:-1] + (0,))
        return e, n, unsampled

    def write_replica_thermodynamic_states(self, state_indices, iteration):
        self._write_record('states', iteration, state_indices)

    def read_replica_thermodynamic_states(self, iteration=slice(None)):
        return self._read_record('states', iteration).astype(np.int64)

    def write_volumes(self, volumes, iteration):
        """Box volume (nm^3) of every replica at this iteration: the reference's 'volumes' f8[iteration, replica]
        (multistatereporter.py:1640-1651), written by constant-pressure runs."""
        self._write_record('volumes', iteration, volumes)

    def read_volumes(self, iteration=slice(None)):
        return self._read_record('volumes', iteration)

    def write_mixing_statistics(self, n_accepted_matrix, n_proposed_matrix, iteration):
        self._write_record('accepted', iteration, n_accepted_matrix)
        self._write_record('proposed', iteration, n_proposed_matrix)

    def read_mixing_statistics(self, iteration=slice(None)):
        return self._read_record('accepted', iteration), self._read_record('proposed', iteration)

    def write_last_iteration(self, last_iteration):
        """The commit marker: everything up to this iteration is complete (multistatereporter.py:1184-1201): the data files
        written since the last marker are synced first, then the marker is replaced atomically."""
        for path in sorted(self._dirty):
            fd = os.open(path, os.O_RDONLY)
            try:
                os.fsync(fd)
            finally:
                os.close(fd)
        self._dirty.clear()
        tmp = os.path.join(self._storage, 'analysis', 'last_iteration.tmp')
        with open(tmp, 'w') as f:
            f.write(str(int(last_iteration)))
            f.flush(); os.fsync(f.fileno())
        os.replace(tmp, os.path.join(self._storage, 'analysis', 'last_iteration'))

    def read_last_iteration(self, last_checkpoint=True):
        p = os.path.join(self._storage, 'analysis', 'last_iteration')
        last = int(open(p).read()) if os.path.exists(p) else -1
        if last_checkpoint:
            cps = [c for c in self.read_checkpoint_iterations() if c <= last]
            return cps[-1] if cps else -1
        return last

    # -- online analysis data (reference: write_online_analysis_data / read_online_analysis_data, used by SAMS)
    def write_online_analysis_data(self, iteration, **kwargs):
        """Per-iteration record of each keyword, or -- ``iteration=None`` -- one static record that is overwritten
        (multistatereporter.py:1204-1339)."""
        d = os.path.join(self._storage, 'analysis', 'online')
        os.makedirs(d, exist_ok=True)
        for name, value in kwargs.items():
            a = np.ascontiguousarray(value, dtype=np.float64 if np.asarray(value).dtype.kind == 'f' else np.int64)
            spec = self._meta.setdefault('online', {})
            if name not in spec:
                spec[name] = {'dtype': a.dtype.str, 'shape': list(a.shape)}
                self._write_meta()
            path = os.path.join(d, name + ('.static.bin' if iteration is None else '.bin'))
            with open(path, 'r+b' if os.path.exists(path) else 'w+b') as f:
                f.seek(0 if iteration is None else int(iteration) * a.nbytes)
                f.write(a.tobytes())
            self._dirty.add(path)

    def write_online_data_dynamic_and_static(self, iteration, **kwargs):
        """multistatereporter.py:1341-1351"""
        self.write_online_analysis_data(None, **kwargs)
        self.write_online_analysis_data(iteration, **kwargs)

    @property
    def real_time_statistics_path(self):
        """``<storage stem>_real_time_analysis.yaml`` next to the storage (multistatereporter.py:1353-1379)."""
        directory, name = os.path.split(os.path.normpath(self._storage))
        return os.path.join(directory, os.path.splitext(name)[0] + '_real_time_analysis.yaml')

    def write_current_statistics(self, data):
        """Append one entry to the real-time statistics file, a YAML list with one entry per offline analysis pass
        (multistatereporter.py:1353-1379); the first write of a fresh run truncates it.  Each entry is one line
        ``- {json}``, which is YAML; non-finite numbers are written as YAML's .inf / -.inf / .nan."""
        path = self.real_time_statistics_path
        if self._overwrite_statistics:
            if os.path.exists(path):
                os.remove(path)
            self._overwrite_statistics = False
        line = json.dumps(_jsonable(data), allow_nan=True)
        line = re.sub(r'(?<![\w."])(-?)Infinity\b', r'\1.inf', line)
        line = re.sub(r'(?<![\w."])NaN\b', '.nan', line)
        with open(path, 'a') as f:
            f.write('- ' + line + '\n')

    def read_online_analysis_data(self, iteration, *keys):
        out = {}
        for name in keys:
            spec = self._meta.get('online', {}).get(name)
            if spec is None:
                raise KeyError(name)
            dt = np.dtype(spec['dtype']); shape = tuple(spec['shape'])
            n = int(np.prod(shape)) if shape else 1
            path = os.path.join(self._storage, 'analysis', 'online', name + ('.static.bin' if iteration is None else '.bin'))
            data = np.fromfile(path, dtype=dt)
            data = data[:(data.size // n) * n].reshape((-1,) + shape)
            out[name] = data[0 if iteration is None else iteration]
        return out

    # -- checkpoints
    def _ckpt(self, iteration):
        return os.path.join(self._storage, 'checkpoint', 'ckpt_%09d.npz' % int(iteration))

    def write_sampler_states(self, sampler_states, iteration, extra=None):
        """Positions/velocities/box of every replica on checkpoint iterations, and of the analysis particles at their
        own intervals (multistatereporter.py:664-700, 1670-1730)."""
        if self.wants_analysis_states(iteration):
            self._write_analysis_particles(sampler_states, int(iteration))
        if int(iteration) % self._checkpoint_interval != 0:
            return False
        x = np.stack([s._positions for s in sampler_states])
        have_v = all(s._velocities is not None for s in sampler_states)
        v = np.stack([s._velocities for s in sampler_states]) if have_v else np.zeros((0,))
        boxes = [s._box_vectors for s in sampler_states]
        have_box = all(b is not None for b in boxes)
        b = np.stack(boxes) if have_box else np.zeros((0,))
        tmp = self._ckpt(iteration) + '.tmp.npz'
        np.savez(tmp, positions=x, velocities=v, box_vectors=b, extra=json.dumps(extra or {}))
        os.replace(tmp, self._ckpt(iteration))
        return True

    def _analysis_file(self, what):
        return os.path.join(self._storage, 'analysis', 'particles_' + what + '.bin')

    def _write_analysis_particles(self, sampler_states, it):
        idx = np.array(self._analysis_particle_indices, dtype=np.int64)
        streams = []
        if self._position_interval != 0 and it % self._position_interval == 0:
            streams.append(('positions', np.stack([s._positions[idx] for s in sampler_states]), self._position_interval))
            if all(s._box_vectors is not None for s in sampler_states):
                streams.append(('box_vectors', np.stack([s._box_vectors for s in sampler_states]), self._position_interval))
        if self._velocity_interval != 0 and it % self._velocity_interval == 0 and all(s._velocities is not None for s in sampler_states):
            streams.append(('velocities', np.stack([s._velocities[idx] for s in sampler_states]), self._velocity_interval))
        for what, a, interval in streams:
            a = np.ascontiguousarray(a, dtype=np.float32)          # the reference stores these as float32
            spec = self._meta.setdefault('analysis_particles', {})
            if what not in spec:
                spec[what] = {'shape': list(a.shape), 'interval': interval, 'indices': list(self._analysis_particle_indices)}
                self._write_meta()
            path = self._analysis_file(what)
            with open(path, 'r+b' if os.path.exists(path) else 'w+b') as f:
                f.seek((it // interval) * a.nbytes)
                f.write(a.tobytes())
            self._dirty.add(path)

    def _read_analysis_particles(self, what, it):
        spec = self._meta.get('analysis_particles', {}).get(what)
        if spec is None or it % spec['interval'] != 0:
            return None
        shape = tuple(spec['shape'])
        n = int(np.prod(shape))
        path = self._analysis_file(what)
        rec = it // spec['interval']
        if not os.path.exists(path) or os.path.getsize(path) < (rec + 1) * n * 4:
            return None
        return np.fromfile(path, dtype=np.float32, count=n, offset=rec * n * 4).reshape(shape).astype(np.float64)

    def read_sampler_states(self, iteration, analysis_particles_only=False):
        if analysis_particles_only:
            # the per-iteration streams of the analysis particles (None when there are none, like the reference)
            if isinstance(iteration, (int, np.integer)) and iteration < 0:
                iteration = self.read_last_iteration(last_checkpoint=False) + 1 + int(iteration)
            x = self._read_analysis_particles('positions', int(iteration))
            if x is None:
                return None
            v = self._read_analysis_particles('velocities', int(iteration))
            b = self._read_analysis_particles('box_vectors', int(iteration))
            return [_states.SamplerState(unit.Quantity(x[k], unit.nanometer),
                                         velocities=None if v is None else unit.Quantity(v[k], unit.nanometer / unit.picosecond),
                                         box_vectors=None if b is None else unit.Quantity(b[k], unit.nanometer))
                    for k in range(x.shape[0])]
        if isinstance(iteration, (int, np.integer)) and iteration < 0:
            iteration = self.read_checkpoint_iterations()[iteration]
        if not os.path.exists(self._ckpt(iteration)):
            return None
        d = np.load(self._ckpt(iteration))
        out = []
        for k in range(d['positions'].shape[0]):
            v = d['velocities'][k] if d['velocities'].ndim == 3 else None
            b = d['box_vectors'][k] if d['box_vectors'].ndim == 3 else None
            out.append(_states.SamplerState(unit.Quantity(d['positions'][k], unit.nanometer),
                                            velocities=None if v is None else unit.Quantity(v, unit.nanometer / unit.picosecond),
                                            box_vectors=None if b is None else unit.Quantity(b, unit.nanometer)))
        return out

    def read_checkpoint_extra(self, iteration):
        d = np.load(self._ckpt(iteration))
        return json.loads(str(d['extra']))

    def read_checkpoint_iterations(self):
        d = os.path.join(self._storage, 'checkpoint')
        its = sorted(int(f[5:14]) for f in os.listdir(d) if f.startswith('ckpt_') and f.endswith('.npz') and '.tmp' not in f)
        return its


class _RestrictedUnpickler(pickle.Unpickler):
    """The object files of a storage directory hold thermodynamic states and MCMC moves of THIS package (plus numpy arrays
    and plain containers).  Nothing else is ever constructed while reading them: a storage directory that names any other
    class is rejected instead of executed (the reference serialises through YAML for the same reason)."""
    _NUMPY_OK = {('numpy.core.multiarray', '_reconstruct'), ('numpy._core.multiarray', '_reconstruct'),
                 ('numpy', 'ndarray'), ('numpy', 'dtype'), ('numpy.core.multiarray', 'scalar'),
                 ('numpy._core.multiarray', 'scalar'), ('numpy._core.numeric', '_frombuffer'),
                 ('numpy.core.numeric', '_frombuffer')}
    _BUILTINS_OK = {'set', 'frozenset', 'tuple', 'list', 'dict', 'complex', 'slice', 'range', 'bytearray', 'object'}

    def find_class(self, module, name):
        if module == 'openmmtools_b200' or module.startswith('openmmtools_b200.'):
            return super().find_class(module, name)
        if (module, name) in self._NUMPY_OK:
            return super().find_class(module, name)
        if module == 'builtins' and name in self._BUILTINS_OK:
            return super().find_class(module, name)
        if module == 'collections' and name in ('OrderedDict', 'defaultdict'):
            return super().find_class(module, name)
        if module == 'copyreg' and name == '_reconstructor':
            return super().find_class(module, name)
        raise pickle.UnpicklingError('storage object file refers to %s.%s, which is not part of a sampler description'
                                     % (module, name))


def _restricted_load(f):
    return _RestrictedUnpickler(f).load()


def _jsonable(x):
    if isinstance(x, dict):
        return {str(k): _jsonable(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_jsonable(v) for v in x]
    if isinstance(x, np.ndarray):
        return _jsonable(x.tolist())
    if isinstance(x, (np.integer,)):
        return int(x)
    if isinstance(x, (np.floating,)):
        return float(x)
    if isinstance(x, unit.Quantity):
        return {'__quantity__': _jsonable(np.asarray(x._md()).tolist()), 'unit_md': str(x.unit)}
    if isinstance(x, (str, int, float, bool)) or x is None:
        return x
    return repr(x)
