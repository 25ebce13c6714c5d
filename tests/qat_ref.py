"""The oracle's restatement of one case of ``tests/golden/qat.npz`` (the learnable quantizers in a train-mode step), shared
by the CPU pin of the restatement and the GPU replay of the fixture."""
import numpy as np

from oracle import qdq as oqdq

GRAD_KEYS = {"scale": "_gscale", "zero_point": "_gzp", "alpha": "_galpha"}  # oracle gradient name -> fixture suffix


def case_geometry(g, name):
    """(qtype, scheme, target, layout, qmin, qmax, ch_axis, per_channel, bit) of a fixture case."""
    qtype, scheme, target, layout = (str(v) for v in g[name + "_cfg"])
    qmin, qmax, ch_axis, perch, _, bit = (int(v) for v in g[name + "_meta"])
    return qtype, scheme, target, layout or "NCHW", qmin, qmax, ch_axis, bool(perch), bit


def oracle_case(g, name, x=None, gy=None, **params):
    """(y, gx, {param: (grad, l1)}) of ``oracle.qdq`` for a fixture case; ``x`` / ``gy`` / parameters default to the
    recorded ones (``scale``, ``zero_point``, ``alpha``)."""
    qtype, _, _, _, qmin, qmax, ch_axis, perch, _ = case_geometry(g, name)
    x = g[name + "_x"] if x is None else x
    gy = g[name + "_gy"] if gy is None else gy
    if qtype == "pact":
        return oqdq.pact_grads(x, params.get("alpha", g[name + "_alpha"]), gy, qmin, qmax)
    s = params.get("scale", g[name + "_scale"])
    zp = params.get("zero_point", g[name + "_zp"])
    if qtype == "dorefa":
        return oqdq.dorefa_grads(x, s, zp, gy, qmin, qmax, ch_axis)
    if qtype == "uniform":
        gx, _, _ = oqdq.ste_backward(x, s, zp, gy, qmin, qmax, ch_axis)
        return oqdq.qdq(x, s, zp, qmin, qmax, ch_axis), gx, {}
    return oqdq.lsq_grads(x, s, zp, gy, qmin, qmax, ch_axis if perch else None,
                          learn_zero_point=qtype == "lsq+" and not perch)


def plant_grid_edges(x, s, zp, qmin, qmax, ch_axis=None):
    """In place: rounding ties (k + 0.5)·s and values landing exactly on qmin / qmax (and half a step beyond them) at the
    head of every quantisation row of ``x`` (the whole tensor per tensor, each channel along ``ch_axis`` per channel) --
    the planting of tests/golden/make_golden.py:gen_qat."""
    rows = x.reshape(1, -1) if ch_axis is None else np.moveaxis(x, ch_axis, 0)
    s, zp = np.asarray(s, np.float32).reshape(-1), np.rint(np.asarray(zp, np.float32).reshape(-1))
    for c in range(rows.shape[0]):
        sc, z = s[min(c, s.size - 1)], zp[min(c, zp.size - 1)]
        units = [0.5, 1.5, -2.5, qmax - z - 0.5, qmin - z + 0.5, qmax - z, qmin - z, qmax - z + 0.5, qmin - z - 0.5]
        for i, u in enumerate(units[:rows[c].size]):
            rows[c].flat[i] = np.float32(u) * sc
    return x


def plant_pact_bounds(x, alpha, signed, at=9):
    """In place: x exactly on the clamp bounds and one ulp either side of each, from flat index ``at`` (as many as fit)."""
    a = np.float32(alpha)
    lo = -a if signed else np.float32(0)
    bounds = [a, np.nextafter(a, np.float32(0)), np.nextafter(a, np.float32(np.inf)), lo,
              np.nextafter(lo, np.float32(-np.inf)), np.nextafter(lo, np.float32(np.inf))]
    flat = x.reshape(-1)
    flat[at:at + len(bounds)] = bounds[:max(0, flat.size - at)]
    return x


def within_l1(got, want, l1, rel=1e-5):
    """|got - want| <= rel * L1 elementwise, L1 the norm of the terms summed into the gradient: any summation order of
    n fp32 terms stays within (n - 1) u L1 of the exact sum, and the orders used (fp64, pairwise, tree reductions)
    stay far below 1e-5 L1 (u = 2^-24, log2(n) << 168 levels)."""
    got, want, l1 = (np.asarray(v, np.float64).reshape(-1) for v in (got, want, l1))
    return got.shape == want.shape and bool(np.all(np.abs(got - want) <= rel * l1))
