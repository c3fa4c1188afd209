"""Minimal host-side plumbing for multi-process runs (one process per GPU).

Only small control messages cross here (the 128-byte NCCL unique id, a seed); all bulk traffic is NCCL inside the
engine.  ``torch.distributed`` is used when it is already initialised (torchrun), otherwise a tiny TCP
exchange on MASTER_ADDR:MASTER_PORT+1.  Replaces the role of mpiplus' bcast
(/root/reference/openmmtools/multistate/replicaexchange.py:255).
"""
import os
import socket
import time


class TorchCommunicator:
    def __init__(self):
        import torch.distributed as dist
        self.dist = dist
        self.rank = dist.get_rank()
        self.world_size = dist.get_world_size()

    def bcast_bytes(self, data, n):
        import torch
        t = torch.zeros(n, dtype=torch.uint8)
        if self.rank == 0:
            t = torch.tensor(list(data[:n].ljust(n, b'\0')), dtype=torch.uint8)
        if self.dist.get_backend() == 'nccl':
            t = t.cuda()
        self.dist.broadcast(t, 0)
        return bytes(t.cpu().tolist())

    def barrier(self):
        self.dist.barrier()

    def gather_object(self, obj):
        """List of every rank's object on rank 0, None elsewhere (checkpoint gather; small control-plane traffic)."""
        out = [None] * self.world_size if self.rank == 0 else None
        self.dist.gather_object(obj, out, dst=0)
        return out


class SocketCommunicator:
    """Rank 0 listens; the others connect and receive.  Enough for a broadcast of a few bytes."""

    def __init__(self):
        self.rank = int(os.environ.get('RANK', '0'))
        self.world_size = int(os.environ.get('WORLD_SIZE', '1'))
        self.addr = os.environ.get('MASTER_ADDR', '127.0.0.1')
        self.port = int(os.environ.get('MASTER_PORT', '29500')) + 1

    def bcast_bytes(self, data, n):
        if self.world_size == 1:
            return data
        if self.rank == 0:
            srv = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
            srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
            srv.bind((self.addr, self.port))
            srv.listen(self.world_size)
            for _ in range(self.world_size - 1):
                c, _a = srv.accept()
                c.sendall(data[:n].ljust(n, b'\0'))
                c.close()
            srv.close()
            return data[:n].ljust(n, b'\0')
        for _ in range(600):
            try:
                c = socket.create_connection((self.addr, self.port), timeout=5)
                break
            except OSError:
                time.sleep(0.1)
        else:
            raise RuntimeError('could not reach rank 0')
        buf = b''
        while len(buf) < n:
            chunk = c.recv(n - len(buf))
            if not chunk:
                break
            buf += chunk
        c.close()
        return buf

    def barrier(self):
        self.bcast_bytes(b'x', 1)

    def gather_object(self, obj):
        """Gather every rank's sampler-state shard -- a list of (replica index, positions, velocities | None, potential |
        None, kinetic | None) -- on rank 0.  The wire format is a fixed binary layout of numbers and raw float64 buffers
        (no pickle: nothing that arrives on the socket is ever executed), sizes and the sender's rank are validated."""
        import struct
        if self.world_size == 1:
            return [obj]
        if self.rank == 0:
            srv = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
            srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
            srv.bind((self.addr, self.port + 1))
            srv.listen(self.world_size)
            out = [None] * self.world_size
            out[0] = obj
            for _ in range(self.world_size - 1):
                c, _a = srv.accept()
                c.settimeout(60)
                r, n = struct.unpack('<iq', _recv_exact(c, 12))
                if not (1 <= r < self.world_size) or out[r] is not None or not (0 <= n <= _MAX_SHARD_BYTES):
                    c.close()
                    srv.close()
                    raise RuntimeError('gather: malformed header from a peer (rank %d, %d bytes)' % (r, n))
                out[r] = _decode_shard(_recv_exact(c, n))
                c.close()
            srv.close()
            return out
        payload = _encode_shard(obj)
        for _ in range(600):
            try:
                c = socket.create_connection((self.addr, self.port + 1), timeout=5)
                break
            except OSError:
                time.sleep(0.1)
        else:
            raise RuntimeError('could not reach rank 0')
        c.sendall(struct.pack('<iq', self.rank, len(payload)) + payload)
        c.close()
        return None


_MAX_SHARD_BYTES = 1 << 34


def _recv_exact(c, n):
    buf = bytearray()
    while len(buf) < n:
        chunk = c.recv(min(1 << 20, n - len(buf)))
        if not chunk:
            raise RuntimeError('gather: connection closed after %d of %d bytes' % (len(buf), n))
        buf += chunk
    return bytes(buf)


_NPT_RECORD = 7   # box edges (3), barostat volume_scale, step, n_attempted, n_accepted


def _encode_shard(shard):
    """[(k, x[N,3], v[N,3] | None, pe | None, ke | None[, npt | None]), ...] -> bytes: count, then per item
    <i k><i n_atoms><B has_v><B has_pe><B has_ke><B has_npt><d pe><d ke> + x (+ v) (+ npt) as little-endian float64.
    npt: a constant-pressure replica's box edges and barostat state, 7 float64 (the counters are exact in float64)."""
    import struct
    import numpy as np
    parts = [struct.pack('<i', len(shard))]
    for item in shard:
        k, x, v, pe, ke = item[:5]
        npt = item[5] if len(item) > 5 else None
        x = np.ascontiguousarray(x, dtype='<f8')
        parts.append(struct.pack('<iiBBBBdd', int(k), x.shape[0], v is not None, pe is not None, ke is not None,
                                 npt is not None, 0.0 if pe is None else float(pe), 0.0 if ke is None else float(ke)))
        parts.append(x.tobytes())
        if v is not None:
            parts.append(np.ascontiguousarray(v, dtype='<f8').tobytes())
        if npt is not None:
            npt = np.ascontiguousarray(npt, dtype='<f8')
            if npt.shape != (_NPT_RECORD,):
                raise ValueError('the constant-pressure record of a replica holds %d numbers' % _NPT_RECORD)
            parts.append(npt.tobytes())
    return b''.join(parts)


def _decode_shard(buf):
    import struct
    import numpy as np
    if len(buf) < 4:
        raise RuntimeError('gather: malformed shard')
    (count,), off = struct.unpack_from('<i', buf, 0), 4
    if count < 0 or count > 1 << 24:
        raise RuntimeError('gather: malformed shard')
    out = []
    for _ in range(count):
        if off + struct.calcsize('<iiBBBBdd') > len(buf):
            raise RuntimeError('gather: malformed shard')
        k, n, hv, hp, hk, hn, pe, ke = struct.unpack_from('<iiBBBBdd', buf, off)
        off += struct.calcsize('<iiBBBBdd')
        nb = n * 24
        if n < 0 or off + nb * (2 if hv else 1) + (8 * _NPT_RECORD if hn else 0) > len(buf):
            raise RuntimeError('gather: malformed shard')
        x = np.frombuffer(buf, dtype='<f8', count=3 * n, offset=off).reshape(n, 3).copy()
        off += nb
        v = None
        if hv:
            v = np.frombuffer(buf, dtype='<f8', count=3 * n, offset=off).reshape(n, 3).copy()
            off += nb
        npt = None
        if hn:
            npt = np.frombuffer(buf, dtype='<f8', count=_NPT_RECORD, offset=off).copy()
            off += 8 * _NPT_RECORD
        out.append((k, x, v, pe if hp else None, ke if hk else None, npt))
    return out


_MAX_EXACT_COUNT = 1 << 53


def sum_counts(comm, counts):
    """The element-wise sum over the ranks of every rank's non-negative integer array `counts` (the same shape everywhere),
    on rank 0; None on the other ranks.  Every rank takes part.  The array travels as the position rows of a one-record
    shard, the format both communicators carry; float64 holds every count below 2**53 exactly, and larger ones are refused
    rather than rounded."""
    import numpy as np
    a = np.ascontiguousarray(counts, np.int64)
    if a.size and (a.min() < 0 or a.max() >= _MAX_EXACT_COUNT):
        raise ValueError('sum_counts: counts must lie in [0, 2**53)')
    flat = a.ravel().astype(np.float64)
    rows = np.concatenate([flat, np.zeros(-flat.size % 3)]).reshape(-1, 3)
    parts = comm.gather_object([(comm.rank, rows, None, None, None)])
    if parts is None:
        return None
    total = np.zeros(a.size, np.int64)
    for part in parts:
        rec = np.asarray(part[0][1], np.float64).ravel()
        if len(part) != 1 or rec.size != rows.size:
            raise RuntimeError('sum_counts: a rank sent a record of another size')
        total += rec[:a.size].astype(np.int64)
    return total.reshape(a.shape)


def default_communicator():
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return TorchCommunicator()
    except ImportError:
        pass
    return SocketCommunicator()
