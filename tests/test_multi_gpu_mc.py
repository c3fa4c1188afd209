"""Monte Carlo move counts over several ranks.  CPU (two processes): _dist.sum_counts adds every rank's counts on rank 0
through both communicators (torch.distributed/gloo and the socket fallback).  GPU (marked gpu, needs >= 2 devices): two
ranks running YANK's SequenceMove reproduce one GPU's trajectory and its move statistics."""
import os
import subprocess
import sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

COUNTS_WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
import numpy as np
from openmmtools_b200 import _dist
if %(gloo)r:
    import torch.distributed as dist
    dist.init_process_group('gloo')
    comm = _dist.TorchCommunicator()
else:
    comm = _dist.SocketCommunicator()
r = comm.rank
counts = np.array([[[3, 0, 7, 1], [5 + r, 0, 0, 2 ** 52 + r]], [[9, 1, 7, 1], [6, 2 * r, 0, 2 ** 52]]], np.int64)
total = _dist.sum_counts(comm, counts)
if r == 0:
    want = 2 * counts + np.array([[[0, 0, 0, 0], [1, 0, 0, 1]], [[0, 0, 0, 0], [0, 2, 0, 0]]])
    assert total.dtype == np.int64 and np.array_equal(total, want), total
else:
    assert total is None
print('ok', r)
'''


@pytest.mark.parametrize('gloo', [True, False])
def test_counts_are_summed_over_two_ranks(tmp_path, gloo):
    script = tmp_path / 'c.py'
    script.write_text(COUNTS_WORKER % {'root': ROOT, 'gloo': gloo})
    if gloo:
        r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                            '--master-addr', '127.0.0.1', '--master-port', '29571', str(script)],
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        assert r.stdout.count('ok') == 2
        return
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE='2', MASTER_ADDR='127.0.0.1', MASTER_PORT='29575')
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    outs = [p.communicate(timeout=120)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert sum(o.count('ok') for o in outs) == 2


def test_counts_beyond_float64_precision_are_refused():
    from openmmtools_b200 import _dist
    with pytest.raises(ValueError):
        _dist.sum_counts(_dist.SocketCommunicator(), np.array([2 ** 53]))


GPU_WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, 'tests'))
import numpy as np
import torch.distributed as dist
dist.init_process_group('gloo')
from test_gpu_mc_moves import yank_sampler
from openmmtools_b200._dist import TorchCommunicator
s = yank_sampler(None, seed=321, communicator=TorchCommunicator())
s.run(3)
s._pull_mc_statistics()
stats = np.array([[[m['n_accepted'], m['n_proposed']] for m in mv.statistics[:2]] for mv in s._mcmc_moves])
np.savez(%(out)r + '_%%d.npz' %% dist.get_rank(), perm=s._replica_thermodynamic_states, u=s._energy_thermodynamic_states,
         x=s._engine.get_positions(), k0=s._engine.k0, stats=stats)
dist.barrier()
'''


def _two_devices():
    import ctypes
    try:
        cuda = ctypes.CDLL('libcudart.so.12')
    except OSError:
        cuda = ctypes.CDLL('libcudart.so')
    n = ctypes.c_int()
    cuda.cudaGetDeviceCount(ctypes.byref(n))
    return n.value >= 2


@pytest.mark.gpu
def test_two_gpus_reproduce_single_gpu_with_mc_moves(tmp_path):
    if not _two_devices():
        pytest.skip('needs 2 GPUs')
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from test_gpu_mc_moves import yank_sampler
    s = yank_sampler(None, seed=321)
    s.run(3)
    s._pull_mc_statistics()
    stats = np.array([[[m['n_accepted'], m['n_proposed']] for m in mv.statistics[:2]] for mv in s._mcmc_moves])
    u1, p1, x1 = s._energy_thermodynamic_states.copy(), s._replica_thermodynamic_states.copy(), s._engine.get_positions()
    script = tmp_path / 'g.py'
    out = str(tmp_path / 'res')
    script.write_text(GPU_WORKER % {'root': ROOT, 'out': out})
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
                        '--master-addr', '127.0.0.1', '--master-port', '29572', str(script)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    d0 = np.load(out + '_0.npz')
    assert np.array_equal(d0['stats'], stats)       # rank 0 holds the totals over both ranks
    for rank in range(2):
        d = np.load(out + '_%d.npz' % rank)
        assert np.array_equal(d['perm'], p1) and np.array_equal(d['u'], u1)
        k0 = int(d['k0'])
        assert np.array_equal(d['x'], x1[k0:k0 + d['x'].shape[0]])
