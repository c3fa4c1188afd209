"""Time the device MBAR passes (rx_mbar_evaluate) against the numpy MBAR of oracle/mbar.py.

For each (K, N): one rx_mbar_create, warm-up, then the median wall time of `--repeats` calls of rx_mbar_evaluate with and
without the Hessian (each call ends in a stream synchronise), a full MBAR solve, and one numpy evaluate of the same
quantities.  Bytes per pass are the algorithmic reads of u_kn: pass 1 reads it once, the row sums once more, the Gram
pass reads both 64-row tiles of each upper tile pair (one for a diagonal pair).  Prints one JSON line per size, with the
card's name and power limit.
Usage: python tools/run_mbar.py [--sizes 256x512000,512x1024000] [--repeats 5] [--no-oracle]"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
import os

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmmtools_b200 import _lib  # noqa: E402
from openmmtools_b200.multistate.mbar import MBAR  # noqa: E402
from oracle import mbar as om  # noqa: E402


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the timing itself needs no nvidia-smi
        return 'unknown (%s)' % e


def pass_bytes(K, N):
    tiles = (K + 63) // 64
    rows_gram = 0
    for i in range(tiles):
        for j in range(i, tiles):
            rows_gram += min(64, K - 64 * i) + (0 if i == j else min(64, K - 64 * j))
    u = 8 * K * N
    return {'logden': u, 'rowsum': u + 8 * N, 'gram': 8 * rows_gram * N + 8 * N}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='256x512000,512x1024000')
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--no-oracle', action='store_true')
    args = ap.parse_args()
    lib = _lib.load()
    for spec in args.sizes.split(','):
        K, N = (int(x) for x in spec.split('x'))
        rng = np.random.default_rng(K)
        N_k = np.full(K, N // K, np.int64)
        N_k[0] += N - N_k.sum()
        u = np.ascontiguousarray(np.linspace(0, 4, K)[:, None] + rng.normal(0, 1, (K, N)))
        f = rng.normal(0, 0.1, K)
        h = C.c_void_p()
        rc = lib.rx_mbar_create(K, N, _ptr(u), _ptr(N_k), C.byref(h))
        if rc:
            raise SystemExit('rx_mbar_create: %s' % lib.rx_mbar_last_error(None).decode())
        s, g, H = C.c_double(), np.empty(K), np.empty((K, K))
        times = {}
        for name, hp in (('evaluate_with_hessian', _ptr(H)), ('evaluate_gradient_only', None)):
            for _ in range(2):
                assert lib.rx_mbar_evaluate(h, _ptr(f), C.byref(s), _ptr(g), hp) == 0
            ts = []
            for _ in range(args.repeats):
                t = time.perf_counter()
                assert lib.rx_mbar_evaluate(h, _ptr(f), C.byref(s), _ptr(g), hp) == 0
                ts.append(time.perf_counter() - t)
            times[name] = float(np.median(ts))
        lib.rx_mbar_destroy(h)
        t = time.perf_counter()
        m = MBAR(u, N_k)
        r = m.compute_free_energy_differences()
        solve_s = time.perf_counter() - t
        iters = m.n_iterations
        m.close()
        out = {'K': K, 'N': N, 'card': card(), 'seconds': times, 'bytes_per_pass': pass_bytes(K, N),
               'solve_seconds_incl_upload_and_covariance': solve_s, 'solve_iterations': iters,
               'dDelta_f_0_last': float(r['dDelta_f'][0, -1])}
        b = out['bytes_per_pass']
        out['achieved_GBps_gradient_only'] = (b['logden'] + b['rowsum']) / times['evaluate_gradient_only'] / 1e9
        if not args.no_oracle:
            t = time.perf_counter()
            om.evaluate(u, N_k, f)
            out['oracle_evaluate_seconds'] = time.perf_counter() - t
            out['speedup_evaluate_with_hessian'] = out['oracle_evaluate_seconds'] / times['evaluate_with_hessian']
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
