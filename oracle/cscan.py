"""ctypes front-end of the C oracle (oracle/csrc/scan_ref.c).  TEST INFRASTRUCTURE ONLY.

Restates the reference's selective_scan_ref
(Mamba/kernels/selective_scan/test_selective_scan.py:168-234) as a plain-C
sequential recurrence so that full-size cases finish in seconds on the CPU.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboracle_scan.so")
_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "csrc", "scan_ref.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "all"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
        _lib.scan_ref_set_threads(int(host_threads()))  # default: physical cores within the quota, not every SMT thread
    return _lib


def set_threads(n: int):
    lib().scan_ref_set_threads(int(n))


def host_threads() -> int:
    """CPU threads for the oracle: PHYSICAL cores inside this process's scheduler affinity mask (cpusets / taskset), capped by the
    cgroup CPU quota -- on a GPU host with many SMT threads and a small CPU quota, one OpenMP thread per logical CPU runs the oracle
    ~100x slower."""
    import os
    try:
        aff = os.sched_getaffinity(0)
    except AttributeError:
        return os.cpu_count() or 1
    cores, cur = set(), {}
    try:
        for line in open("/proc/cpuinfo"):
            if ":" in line:
                k, v = line.split(":", 1)
                cur[k.strip()] = v.strip()
            elif cur:
                if int(cur.get("processor", -1)) in aff:
                    cores.add((cur.get("physical id"), cur.get("core id")))
                cur = {}
    except OSError:
        pass
    n = len(cores) if cores else len(aff)
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(q) // int(per)))
    except (OSError, ValueError):
        pass
    return max(1, min(n, len(aff)))


def use_host_threads() -> int:
    """size the OpenMP scan and torch's intra-op pool for the CPU oracle; returns the thread count"""
    n = host_threads()
    set_threads(n)
    torch.set_num_threads(n)
    return n


def _f32(t):
    if t is None:
        return None
    return np.ascontiguousarray(t.detach().to(torch.float32).cpu().numpy())


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _shapes(u, A, B):
    b, D, L = u.shape
    N = A.shape[1]
    G = B.shape[1] if B.dim() == 4 else 1
    return b, D, L, N, G


def scan_fwd(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False,
             fp64=False, return_last_state=False):
    """Sequential oracle forward. Inputs: torch tensors (any float dtype, cast to fp32
    first exactly like the reference does with .float()).  Returns fp32 (or fp64) torch tensor."""
    b, Dm, L, N, G = _shapes(u, A, B)
    un, dn, An, Bn, Cn, Dn, bn = map(_f32, (u, delta, A, B, C, D, delta_bias))
    if fp64:
        out = np.empty((b, Dm, L), np.float64)
        lib().scan_ref_fwd_f64(_p(un), _p(dn), _p(An), _p(Bn), _p(Cn), _p(Dn), _p(bn),
                               int(delta_softplus), _p(out), b, Dm, L, N, G)
        return torch.from_numpy(out)
    out = np.empty((b, Dm, L), np.float32)
    last = np.empty((b, Dm, N), np.float32) if return_last_state else None
    lib().scan_ref_fwd_f32(_p(un), _p(dn), _p(An), _p(Bn), _p(Cn), _p(Dn), _p(bn),
                           int(delta_softplus), _p(out), _p(last), b, Dm, L, N, G)
    o = torch.from_numpy(out)
    return (o, torch.from_numpy(last)) if return_last_state else o


def scan_bwd(u, delta, A, B, C, D, delta_bias, dout, delta_softplus=False):
    """Analytic fp64 backward. Returns (du, ddelta, dA, dB, dC, dD, dbias) as fp64 tensors."""
    b, Dm, L, N, G = _shapes(u, A, B)
    un, dn, An, Bn, Cn, Dn, bn, gn = map(_f32, (u, delta, A, B, C, D, delta_bias, dout))
    du = np.zeros((b, Dm, L)); dd = np.zeros((b, Dm, L)); dA = np.zeros((Dm, N))
    dB = np.zeros((b, G, N, L)); dC = np.zeros((b, G, N, L))
    dD = np.zeros((Dm,)) if D is not None else None
    db = np.zeros((Dm,)) if delta_bias is not None else None
    lib().scan_ref_bwd_f64(_p(un), _p(dn), _p(An), _p(Bn), _p(Cn), _p(Dn), _p(bn),
                           int(delta_softplus), _p(gn), _p(du), _p(dd), _p(dA), _p(dB), _p(dC),
                           _p(dD), _p(db), b, Dm, L, N, G)
    t = lambda a: None if a is None else torch.from_numpy(a)
    return tuple(map(t, (du, dd, dA, dB, dC, dD, db)))


class Scan(torch.autograd.Function):
    """The sequential oracle as a differentiable function: Scan.apply(u, delta, A, B, C, D, delta_bias, delta_softplus).
    float64 inputs run scan_fwd(fp64=True) / scan_bwd, any other dtype scan_fwd / scan_bwd_f32.  The group count comes from B.shape as
    in _shapes; results (output and gradients) come back in u's dtype and on u's device, gradients shaped like their inputs, None for an
    absent D or delta_bias.  The C oracle reads fp32 inputs: a float64 caller's inputs and incoming gradient are rounded to fp32
    (relative 6e-8) before the float64 recurrence."""

    @staticmethod
    def forward(ctx, u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False):
        ctx.save_for_backward(u, delta, A, B, C, D, delta_bias)
        ctx.delta_softplus = delta_softplus
        out = scan_fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, fp64=u.dtype == torch.float64)
        return out.to(device=u.device, dtype=u.dtype)

    @staticmethod
    def backward(ctx, dout):
        ins = ctx.saved_tensors
        bwd = scan_bwd if ins[0].dtype == torch.float64 else scan_bwd_f32
        grads = bwd(*ins, dout, ctx.delta_softplus)
        return tuple(None if g is None else g.view(t.shape).to(device=t.device, dtype=t.dtype) for g, t in zip(grads, ins)) + (None,)


def scan_fwd_mag(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False):
    """scan_fwd(fp64=True) and the magnitude S of every output (oracle/scan_bound.py) -> (out, S), float64 torch tensors"""
    b, Dm, L, N, G = _shapes(u, A, B)
    un, dn, An, Bn, Cn, Dn, bn = map(_f32, (u, delta, A, B, C, D, delta_bias))
    out, S = np.empty((b, Dm, L), np.float64), np.empty((b, Dm, L), np.float64)
    lib().scan_ref_fwd_mag(_p(un), _p(dn), _p(An), _p(Bn), _p(Cn), _p(Dn), _p(bn), int(delta_softplus), _p(out), _p(S),
                           b, Dm, L, N, G)
    return torch.from_numpy(out), torch.from_numpy(S)


def _bwd_outputs(b, Dm, L, N, G, has_D, has_bias, dt):
    return [np.zeros((b, Dm, L), dt), np.zeros((b, Dm, L), dt), np.zeros((Dm, N), dt), np.zeros((b, G, N, L), dt),
            np.zeros((b, G, N, L), dt), np.zeros((Dm,), dt) if has_D else None, np.zeros((Dm,), dt) if has_bias else None]


def _t(a):
    return None if a is None else torch.from_numpy(a)


def scan_bwd_mag(u, delta, A, B, C, D, delta_bias, dout, delta_softplus=False):
    """scan_bwd and the magnitude S of every gradient -> ((du, ddelta, dA, dB, dC, dD, dbias), (S_du, ..., S_dbias)), float64"""
    b, Dm, L, N, G = _shapes(u, A, B)
    un, dn, An, Bn, Cn, Dn, bn, gn = map(_f32, (u, delta, A, B, C, D, delta_bias, dout))
    g = _bwd_outputs(b, Dm, L, N, G, D is not None, delta_bias is not None, np.float64)
    s = _bwd_outputs(b, Dm, L, N, G, D is not None, delta_bias is not None, np.float64)
    lib().scan_ref_bwd_mag(_p(un), _p(dn), _p(An), _p(Bn), _p(Cn), _p(Dn), _p(bn), int(delta_softplus), _p(gn),
                           *map(_p, g), *map(_p, s), b, Dm, L, N, G)
    return tuple(map(_t, g)), tuple(map(_t, s))


def scan_bwd_f32(u, delta, A, B, C, D, delta_bias, dout, delta_softplus=False):
    """the analytic backward evaluated sequentially in fp32 -> (du, ddelta, dA, dB, dC, dD, dbias), float32"""
    b, Dm, L, N, G = _shapes(u, A, B)
    un, dn, An, Bn, Cn, Dn, bn, gn = map(_f32, (u, delta, A, B, C, D, delta_bias, dout))
    g = _bwd_outputs(b, Dm, L, N, G, D is not None, delta_bias is not None, np.float32)
    lib().scan_ref_bwd_f32(_p(un), _p(dn), _p(An), _p(Bn), _p(Cn), _p(Dn), _p(bn), int(delta_softplus), _p(gn),
                           *map(_p, g), b, Dm, L, N, G)
    return tuple(map(_t, g))
