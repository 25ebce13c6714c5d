"""Generate ``tests/golden/ref_ext.npz``: outputs of the reference's own CUDA extensions on the inputs that
``tests/test_gpu_reference_ext.py`` builds.  Needs a GPU and the extensions built unmodified from the reference
checkout by ``oracle/build_ref.py`` into ``oracle/_ref/``:

    python oracle/build_ref.py && python tests/golden/make_golden_ref_ext.py [OUT.npz]
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import test_gpu_reference_ext as T  # noqa: E402
from gpu_util import dev, t  # noqa: E402


def load(name):
    path = os.path.join(ROOT, "oracle", "_ref", name + ".so")
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_ext.npz")
    fq, gq = load("fake_quant_ref"), load("gptq_ref")
    out = {}
    for n, qmin, qmax, zp in T.PERTENSOR_CASES:
        key = T.case_key("pt", n, qmin, qmax, zp)
        x, gy, s, z = T.pertensor_inputs(n, qmin, qmax, zp)
        idx = T.sample_index(n, n)
        xt, gt = t(x), t(gy)
        st, zt = t(s).requires_grad_(True), t(z).requires_grad_(True)
        out[key + "_y"] = fq.quant_pertensor_forward(xt, st, zt, qmin, qmax, 0).cpu().numpy()[idx]
        gx, gs, gz = fq.quant_pertensor_backward(xt, st, zt, gt, qmin, qmax, 0)
        out[key + "_gx"], out[key + "_gs"], out[key + "_gz"] = gx.cpu().numpy()[idx], gs.cpu().numpy(), gz.cpu().numpy()
    for shape, ch_axis, qmin, qmax in T.PERCHANNEL_CASES:
        key = T.case_key("pc", shape, ch_axis, qmin, qmax)
        x, gy, s, z = T.perchannel_inputs(shape, ch_axis, qmin, qmax)
        idx = T.sample_index(x.size, sum(shape))
        xt, gt = t(x), t(gy)
        st, zt = t(s).requires_grad_(True), t(z).requires_grad_(True)
        out[key + "_y"] = fq.quant_perchannel_forward(xt, st, zt, qmin, qmax, ch_axis, 0).cpu().numpy().reshape(-1)[idx]
        gx, gs, gz = fq.quant_perchannel_backward(xt, st, zt, gt, qmin, qmax, ch_axis, 0)
        out[key + "_gx"] = gx.cpu().numpy().reshape(-1)[idx]
        out[key + "_gs"], out[key + "_gz"] = gs.cpu().numpy().reshape(-1), gz.cpu().numpy().reshape(-1)
    x, gy, s, z = (v.to(dev()) for v in T.gate_inputs())
    gates = []
    for rs, rz in T.GATE_CASES:
        _, gs, gz = fq.quant_pertensor_backward(x, s.clone().requires_grad_(rs), z.clone().requires_grad_(rz), gy, -8, 7, 0)
        gates.append((float(gs) == 0, float(gz) == 0))
    out["gate_zero"] = np.array(gates, dtype=np.bool_)
    for bit, m, k, n, gs in T.GPTQ_CASES:
        x, qw, scales, zeros, bias, name = T.gptq_inputs(bit, m, k, n, gs)
        y = bias.expand(m, n).contiguous()
        args = (x, qw, y, scales, zeros) + (() if gs == -1 else (gs,))
        getattr(gq, name)(*args)
        out[T.case_key("gptq", bit, m, k, n, gs) + "_y"] = y.cpu().numpy().reshape(-1)[T.sample_index(m * n, bit * 1000 + m)]
    torch.cuda.synchronize()
    np.savez_compressed(out_path, **out)
    print("wrote", out_path, sum(v.nbytes for v in out.values()), "bytes")


if __name__ == "__main__":
    main()
