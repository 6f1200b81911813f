"""Oracles of frequency-decoupled guidance (model_wrapper's fdg_scales) -- TEST INFRASTRUCTURE.

* `fdg_fp64`: diffusers' per-level form in float64 with the same Down / Up: the Laplacian pyramids of c and u,
  u_l + w_l*(c_l - u_l) per level, then the reconstruction G_l = Up(G_{l+1}) + L_l.
* `fdg_exact`: the contract of include/dpm_solver_b200.h in numpy fp32, operation for operation (the correction form
  on the pyramid of d = c - u); the bit-exact reference for dpm_fdg_guided.
* `FDGOracle`: the numpy executor plus `fdg_guided`.
* `guided_net`: a network for the UNMODIFIED reference's guidance_type="uncond" wrapper that runs the real network on
  the doubled batch and returns the FDG output.
"""
import numpy as np
import torch

from tcfg_oracle import TCFGOracle

f32 = np.float32
H_DOWN = [1, 5, 10, 10, 5, 1]           # /32
UP_EVEN = [1, 21, 35, 7]                # /64, taps i-2 .. i+1
UP_ODD = [7, 35, 21, 1]                 # /64, taps i-1 .. i+2


def _refl(j, n):
    j = np.asarray(j)
    return np.where(j < 0, -j, np.where(j > n - 1, 2 * (n - 1) - j, j))


def _down(a, axis, dt):
    """Down along `axis` (even length n -> n/2): sum_k fl(h_k*a[R(2i-2+k)]), left to right, in `dt`."""
    a = np.moveaxis(a, axis, -1)
    n = a.shape[-1]
    i = np.arange(n // 2)
    s = None
    for k, h in enumerate(H_DOWN):
        t = dt(h / 32) * a[..., _refl(2 * i - 2 + k, n)]
        s = t if s is None else s + t
    return np.moveaxis(s, -1, axis)


def _up(a, axis, dt):
    """Up along `axis` (m -> 2m), the polyphase taps of the contract, left to right, in `dt`."""
    a = np.moveaxis(a, axis, -1)
    m = a.shape[-1]
    i = np.arange(m)
    out = np.empty(a.shape[:-1] + (2 * m,), a.dtype)
    for phase, (taps, first) in enumerate(((UP_EVEN, -2), (UP_ODD, -1))):
        s = None
        for k, c in enumerate(taps):
            t = dt(c / 64) * a[..., _refl(i + first + k, m)]
            s = t if s is None else s + t
        out[..., phase::2] = s
    return np.moveaxis(out, -1, axis)


def down2(a, dt=f32):
    return _down(_down(a, -1, dt), -2, dt)        # rows (along W) first, then columns


def up2(a, dt=f32):
    return _up(_up(a, -1, dt), -2, dt)


def _scale_rows(scales, B, levels, dt):
    """[B, levels] scales (one row per sample) from shared scales or per-sample rows."""
    s = scales.detach().cpu().numpy() if torch.is_tensor(scales) else np.asarray(scales)
    s = np.asarray(s, np.float32).astype(dt)
    return np.broadcast_to(s.reshape(-1, levels), (B, levels))


def fdg_exact(c, u, scales, levels):
    """g as dpm_fdg_guided computes it, in c's torch dtype: fp32 arithmetic on the widened outputs, each product
    rounded, sums left to right, then one rounding to the outputs' dtype. `scales`: N numbers or [B, N]."""
    dtype = c.dtype
    cn = c.detach().float().cpu().numpy()
    un = u.detach().float().cpu().numpy()
    B = cn.shape[0]
    w = _scale_rows(scales, B, levels, f32)
    bshape = (B,) + (1,) * (cn.ndim - 1)
    with np.errstate(all="ignore"):
        d = cn - un
        g = un + w[:, 0].reshape(bshape) * d
        if levels > 1:
            G = [d]
            for _ in range(levels - 1):
                G.append(down2(G[-1]))
            delta = [(w[:, l] - w[:, l - 1]).astype(f32).reshape(bshape) for l in range(levels)]
            E = delta[levels - 1] * G[levels - 1]
            for l in range(levels - 2, 0, -1):
                E = delta[l] * G[l] + up2(E)
            g = g + up2(E)
    return torch.from_numpy(np.ascontiguousarray(g, f32)).to(dtype)


def fdg_fp64(c, u, scales, levels):
    """diffusers' per-level form in float64: Laplacian pyramids of c and u, u_l + w_l*(c_l - u_l) per level, then the
    reconstruction. Returns a float64 numpy array."""
    dt = np.float64
    cn = np.asarray(c.double().cpu().numpy() if torch.is_tensor(c) else c, dt)
    un = np.asarray(u.double().cpu().numpy() if torch.is_tensor(u) else u, dt)
    B = cn.shape[0]
    w = _scale_rows(scales, B, levels, dt)
    bshape = (B,) + (1,) * (cn.ndim - 1)

    def lap(x):
        G = [x]
        for _ in range(levels - 1):
            G.append(down2(G[-1], dt))
        return [G[l] - up2(G[l + 1], dt) for l in range(levels - 1)] + [G[-1]]
    Lc, Lu = lap(cn), lap(un)
    L = [Lu[l] + w[:, l].reshape(bshape) * (Lc[l] - Lu[l]) for l in range(levels)]
    g = L[-1]
    for l in range(levels - 2, -1, -1):
        g = up2(g, dt) + L[l]
    return g


class FDGOracle(TCFGOracle):
    """The numpy executor (every model type and guidance form, UniPC included) with dpm_fdg_guided (bit-exact, one
    launch)."""

    def fdg_guided(self, e_cond, e_uncond, scales, levels):
        from dpm_solver_b200 import ops
        ops.fdg_check(e_cond.shape, levels, e_cond.dtype)
        self.launches += 1
        self.log.append(("fdg", 2))
        return fdg_exact(e_cond, e_uncond, scales, levels).to(e_cond.device)


def guided_net(net, uc, c, scales, calls=None):
    """net_g(x, t_input) for a guidance_type="uncond" wrapper: the FDG output of `net` on cat([x, x]) with cat([uc, c]).
    `calls`, when a list, receives one entry per network call."""
    levels = scales.shape[-1] if torch.is_tensor(scales) else len(scales)

    def fn(x, t):
        if calls is not None:
            calls.append(tuple(x.shape))
        out_u, out_c = net(torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c])).chunk(2)
        return fdg_exact(out_c, out_u, scales, levels)
    return fn
