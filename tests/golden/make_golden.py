"""Generate golden vectors by running the UNMODIFIED reference (/root/reference) on CPU.

Run once in the build container (the reference is not present on the GPU box):
    python tests/golden/make_golden.py
Outputs small ``.npz`` fixtures next to this file; they pin ``oracle/`` (tests/test_oracle_golden.py)
and serve as known-answer inputs for the CUDA parity tests (tests/test_gpu_*.py).

Reference entry points exercised (paths relative to /root/reference):
  sparsebit/quantization/quantizers/quant_tensor.py:159-185  ort_fake_quant (CPU branch :181-184)
  sparsebit/quantization/quantizers/quant_tensor.py:128-156  trt_fake_quant (CPU branch :154-155)
  sparsebit/quantization/quantizers/quant_tensor.py:46-71    MySTE.backward (STE backward, Python statement)
  sparsebit/quantization/quantizers/base.py:33-39,66-68      Quantizer.update_observer / calc_qparams
  sparsebit/quantization/observers/{minmax,mse,percentile,kl_histogram}.py
  sparsebit/sparse/sparsers/l1norm.py:14-26                  unstructured mask
  large_language_models/llama/quantization/utils/quant.py    Quantizer.find_params, QuantLinear.pack
  large_language_models/llama/quantization/test_cuda_kernel.py:21-47  known-answer construction
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_import as R  # noqa: E402

R.install_shims()
from sparsebit.quantization.common import Backend  # noqa: E402
from sparsebit.quantization.quantizers import build_quantizer  # noqa: E402
from sparsebit.quantization.quantizers.quant_tensor import ort_fake_quant, trt_fake_quant  # noqa: E402


def save(name, **arrays):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, os.path.getsize(path), "bytes")


def gen_qdq():
    g = torch.Generator().manual_seed(1234)
    out = {}
    cases = []
    specs = [
        # name, shape, qscheme, bit, target, layout
        ("pt_sym8", (2, 3, 9, 7), "per-tensor-symmetric", 8, "feature", "NCHW"),
        ("pt_aff8", (2, 3, 9, 7), "per-tensor-affine", 8, "feature", "NCHW"),
        ("pt_aff4", (5, 37), "per-tensor-affine", 4, "feature", "NCHW"),
        ("pc_w_sym8", (6, 4, 3, 3), "per-channel-symmetric", 8, "weight", None),
        ("pc_w_aff4", (7, 11), "per-channel-affine", 4, "weight", None),
        ("pc_a_nchw_sym8", (2, 5, 7, 7), "per-channel-symmetric", 8, "feature", "NCHW"),
        ("pc_a_nlc_aff8", (3, 5, 8), "per-channel-affine", 8, "feature", "NLC"),
        ("pc_a_nlc_sym8_c7", (2, 6, 7), "per-channel-symmetric", 8, "feature", "NLC"),
    ]
    for name, shape, scheme, bit, target, layout in specs:
        cfg = R.make_cfg(scheme, bit, target, "minmax", layout or "NCHW")
        q = build_quantizer(cfg)
        q.set_backend(Backend.VIRTUAL)
        x = torch.randn(shape, generator=g) * 1.7
        if "aff" in name and target == "feature":
            x = torch.relu(x) + 0.0  # post-ReLU style, affine
        # exact ties and out-of-range values
        flat = x.reshape(-1)
        q.update_observer(x)
        scale, zp = q.calc_qparams()
        s_flat = scale.reshape(-1)
        flat[0] = 0.5 * s_flat[0]
        flat[1] = 1.5 * s_flat[0]
        flat[2] = -2.5 * s_flat[0]
        flat[3] = 1e4
        flat[4] = -1e4
        # fractional zero points (learned LSQ+ style), incl. exact .5 (Q1)
        zp2 = zp.clone()
        if "aff" in name:
            zp2 = zp2 + 0.5
        y = ort_fake_quant(x, scale, zp2, q.qdesc)
        cases.append(name)
        out[name + "_x"] = x.numpy()
        out[name + "_scale"] = scale.reshape(-1).numpy()
        out[name + "_zp"] = zp2.reshape(-1).numpy()
        out[name + "_y"] = y.numpy()
        out[name + "_meta"] = np.array([q.qdesc.qmin, q.qdesc.qmax, q.qdesc.ch_axis, int(q.qdesc.is_perchannel)])
        if "sym" in name:
            yt = trt_fake_quant(x, scale, zp, q.qdesc)
            out[name + "_ytrt"] = yt.numpy()
    out["cases"] = np.array(cases)
    save("qdq", **out)


def gen_observers():
    g = torch.Generator().manual_seed(4321)
    out = {}
    cases = []
    specs = [
        # name, observer, scheme, bit, target, layout, shapes(batches), alpha
        ("minmax_pt_sym", "minmax", "per-tensor-symmetric", 8, "feature", "NCHW", [(2, 3, 8, 8)] * 3, 1e-3),
        ("minmax_pt_aff", "minmax", "per-tensor-affine", 8, "feature", "NCHW", [(2, 3, 8, 8)] * 2, 1e-3),
        ("minmax_pc_w", "minmax", "per-channel-symmetric", 8, "weight", None, [(6, 4, 3, 3)], 1e-3),
        ("minmax_pc_nchw", "minmax", "per-channel-affine", 8, "feature", "NCHW", [(4, 5, 7, 7)], 1e-3),
        ("minmax_pc_nlc", "minmax", "per-channel-symmetric", 8, "feature", "NLC", [(3, 9, 8)], 1e-3),
        ("mse_pt_sym", "mse", "per-tensor-symmetric", 8, "feature", "NCHW", [(2, 3, 16, 16)] * 2, 1e-3),
        ("mse_pt_aff4", "mse", "per-tensor-affine", 4, "feature", "NCHW", [(2, 3, 16, 16)] * 2, 1e-3),
        ("pct_pt_sym", "percentile", "per-tensor-symmetric", 8, "feature", "NCHW", [(4, 3, 16, 16)] * 2, 1e-2),
        ("pct_pt_aff", "percentile", "per-tensor-affine", 8, "feature", "NCHW", [(4, 3, 16, 16)] * 2, 1e-3),
        ("pct_pc_w", "percentile", "per-channel-symmetric", 8, "weight", None, [(5, 64, 3, 3)], 2e-2),
        ("kl_pt_sym", "kl_histogram", "per-tensor-symmetric", 8, "feature", "NCHW", [(2, 3, 16, 16)] * 2, 1e-3),
        ("kl_pt_aff4", "kl_histogram", "per-tensor-affine", 4, "feature", "NCHW", [(2, 3, 16, 16)] * 2, 1e-3),
    ]
    for name, obs, scheme, bit, target, layout, shapes, alpha in specs:
        cfg = R.make_cfg(scheme, bit, target, obs, layout or "NCHW", alpha=alpha)
        q = build_quantizer(cfg)
        q.set_backend(Backend.VIRTUAL)
        xs = []
        for i, shp in enumerate(shapes):
            x = torch.randn(shp, generator=g) * (1.0 + 0.3 * i)
            if "aff" in name and target == "feature":
                x = torch.relu(x)
            xs.append(x)
            q.update_observer(x)
        scale, zp = q.calc_qparams()
        cases.append(name)
        for i, x in enumerate(xs):
            out[f"{name}_x{i}"] = x.numpy()
        out[name + "_nb"] = np.array(len(xs))
        out[name + "_scale"] = scale.reshape(-1).numpy()
        out[name + "_zp"] = zp.reshape(-1).numpy()
        if obs != "mse":
            out[name + "_min"] = q.observer.min_val.reshape(-1).numpy()
            out[name + "_max"] = q.observer.max_val.reshape(-1).numpy()
        out[name + "_meta"] = np.array(
            [q.qdesc.qmin, q.qdesc.qmax, q.qdesc.ch_axis, int(q.qdesc.is_perchannel), int(q.qdesc.is_symmetric), bit]
        )
        out[name + "_alpha"] = np.array(alpha)
    out["cases"] = np.array(cases)
    # torch.histc known answers (ATen CPU), incl. values exactly on edges
    x = torch.randn(5000, generator=g) * 2.0
    am = x.abs().max()
    edges = torch.linspace(-am.item(), am.item(), 2049)
    x[:2049] = edges  # every edge value itself
    x[2049] = am
    x[2050] = -am
    h = torch.histc(x, bins=2048, min=-am.item(), max=am.item())
    out["histc_x"] = x.numpy()
    out["histc_absmax"] = am.numpy()
    out["histc_counts"] = h.numpy()
    out["histc_edges"] = edges.numpy()
    save("observers", **out)


def gen_sparse():
    from sparsebit.sparse.sparsers import build_sparser

    g = torch.Generator().manual_seed(99)
    out = {}
    cases = []
    for name, shape, ratio in [
        ("conv_r50", (8, 4, 3, 3), 0.5),
        ("lin_r25", (10, 33), 0.25),
        ("lin_r75", (10, 33), 0.75),
        ("lin_r100", (6, 5), 1.0),
        ("ties", (4, 16), 0.5),
        ("r0", (3, 5), 0.0),
    ]:
        cfg = R._CfgNode({"SPARSER": {"TYPE": "unstructed", "STRATEGY": "l1norm", "RATIO": ratio}})
        sp = build_sparser(cfg, opr=None)
        w = torch.randn(shape, generator=g)
        if name == "ties":
            w = torch.round(w * 2) / 2  # many equal magnitudes
        mask = sp.calc_mask(w)
        cases.append(name)
        out[name + "_w"] = w.numpy()
        out[name + "_mask"] = mask.numpy()
        out[name + "_masked"] = (w * mask).numpy()
        out[name + "_ratio"] = np.array(ratio)
    out["cases"] = np.array(cases)
    save("sparse", **out)


def gen_gptq():
    # stub the CUDA loader imported by utils/quant.py:5
    qroot = os.path.join(R.REFERENCE_ROOT, "large_language_models/llama/quantization")
    sys.path.insert(0, qroot)
    stub = types.ModuleType("utils.load_cuda_kernel")
    stub.cuda_kernel = None
    sys.modules["utils.load_cuda_kernel"] = stub
    from utils.quant import QuantLinear, Quantizer, quantize  # noqa: E402

    torch.manual_seed(7)
    out = {}
    cases = []
    # (name, B-shape, M(in), N(out), GS) -- scaled-down mirrors of test_cuda_kernel.py:50-126
    for name, bshape, M, N, GS in [
        ("single_block", (1,), 128, 64, -1),
        ("single_irregular", (1,), 127, 61, -1),
        ("irregular_b31", (31,), 333, 251, -1),
        ("tokens_4x8", (4, 8), 256, 96, -1),
        ("group128_b29", (29,), 512, 136, 128),
        ("group384_b4", (4,), 768, 72, 384),
        ("group128_m130", (130,), 256, 128, 128),
    ]:
        layer = torch.nn.Linear(M, N)
        vec = torch.randn(bshape + (M,))
        quantizer = Quantizer()
        quantizer.configure(bit=4, perchannel=True, sym=False, mse=False)
        quantizer.find_params(layer.weight.data, weight=True, groupsize=GS)
        layer.weight.data = quantize(
            layer.weight.data.view(-1, M if GS == -1 else GS),
            quantizer.scale.view(-1, 1),
            quantizer.zero.view(-1, 1),
            quantizer.maxq,
        ).view(N, M)
        w_orig_scale, w_orig_zero = quantizer.scale.clone(), quantizer.zero.clone()
        ql = QuantLinear(M, N, bit=4, groupsize=GS)
        ql.pack(layer, quantizer.scale, quantizer.zero)
        with torch.no_grad():
            gt = layer(vec)
        cases.append(name)
        out[name + "_x"] = vec.numpy()
        out[name + "_wdq"] = layer.weight.data.numpy()
        out[name + "_qweight"] = ql.qweight.numpy()
        out[name + "_scales"] = ql.scales.reshape(N, -1).numpy()
        out[name + "_zeros"] = ql.zeros.reshape(N, -1).numpy()
        out[name + "_zero_int"] = w_orig_zero.reshape(N, -1).numpy()
        out[name + "_bias"] = ql.bias.detach().numpy()
        out[name + "_gt"] = gt.numpy()
        out[name + "_gs"] = np.array(GS)
    out["cases"] = np.array(cases)
    save("gptq", **out)
    # 3-bit / 2-bit rows (SURVEY 8f #3): scaled-down mirrors of the bit=2,3 cases of test_cuda_kernel.py
    out, cases = {}, []
    for name, bit, bshape, M, N, GS in [
        ("b3_single", 3, (1,), 1024, 40, -1),
        ("b3_irregular", 3, (1,), 719, 157, -1),
        ("b3_irregular_b31", 3, (31,), 333, 251, -1),
        ("b3_tokens_4x8", 3, (4, 8), 256, 96, -1),
        ("b3_group128_b29", 3, (29,), 512, 136, 128),
        ("b3_group384_b4", 3, (4,), 768, 40, 384),
        ("b2_single", 2, (1,), 1024, 40, -1),
        ("b2_irregular", 2, (1,), 719, 157, -1),
        ("b2_irregular_b31", 2, (31,), 333, 251, -1),
        ("b2_tokens_4x8", 2, (4, 8), 256, 96, -1),
        ("b2_group64_b29", 2, (29,), 512, 136, 64),
        ("b2_group192_b4", 2, (4,), 768, 40, 192),
    ]:
        layer = torch.nn.Linear(M, N)
        vec = torch.randn(bshape + (M,))
        quantizer = Quantizer()
        quantizer.configure(bit=bit, perchannel=True, sym=False, mse=False)
        quantizer.find_params(layer.weight.data, weight=True, groupsize=GS)
        layer.weight.data = quantize(
            layer.weight.data.view(-1, M if GS == -1 else GS),
            quantizer.scale.view(-1, 1),
            quantizer.zero.view(-1, 1),
            quantizer.maxq,
        ).view(N, M)
        ql = QuantLinear(M, N, bit=bit, groupsize=GS)
        ql.pack(layer, quantizer.scale, quantizer.zero)
        with torch.no_grad():
            gt = layer(vec)
        cases.append(name)
        out[name + "_x"] = vec.numpy()
        out[name + "_wdq"] = layer.weight.data.numpy()
        out[name + "_qweight"] = ql.qweight.numpy()
        out[name + "_scales"] = ql.scales.reshape(N, -1).numpy()
        out[name + "_zeros"] = ql.zeros.reshape(N, -1).numpy()
        out[name + "_zero_int"] = quantizer.zero.reshape(N, -1).numpy()
        out[name + "_bias"] = ql.bias.detach().numpy()
        out[name + "_gt"] = gt.numpy()
        out[name + "_meta"] = np.array([bit, GS])
    out["cases"] = np.array(cases)
    save("gptq_lowbit", **out)


def gen_next_rows():
    """SURVEY 8(f)#2 rows: LSQ / LSQ+ / PACT / DoReFa quantizers and the MovingAverage observer."""
    g = torch.Generator().manual_seed(2024)
    out = {}
    cases = []
    specs = [
        # name, qtype, observer, scheme, bit, target, layout, shapes
        ("lsq_pt_a4", "lsq", "minmax", "per-tensor-affine", 4, "feature", "NCHW", [(4, 3, 12, 12)] * 2),
        ("lsq_pt_sym4", "lsq", "minmax", "per-tensor-symmetric", 4, "feature", "NCHW", [(4, 3, 12, 12)]),
        ("lsq_pc_w4", "lsq", "minmax", "per-channel-symmetric", 4, "weight", None, [(8, 5, 3, 3)]),
        ("lsqp_pt_a8", "lsq+", "minmax", "per-tensor-affine", 8, "feature", "NCHW", [(4, 3, 12, 12)] * 2),
        ("lsqp_pc_w4", "lsq+", "minmax", "per-channel-symmetric", 4, "weight", None, [(8, 5, 3, 3)]),
        ("pact_pt_a4", "pact", "minmax", "per-tensor-affine", 4, "feature", "NCHW", [(4, 3, 12, 12)]),
        ("pact_pt_s8", "pact", "minmax", "per-tensor-symmetric", 8, "feature", "NCHW", [(4, 3, 12, 12)]),
        ("dorefa_w4", "dorefa", "minmax", "per-tensor-symmetric", 4, "weight", None, [(8, 5, 3, 3)]),
        ("mavg_pt", "uniform", "moving_average", "per-tensor-symmetric", 8, "feature", "NCHW", [(5, 3, 8, 8), (4, 3, 8, 8), (6, 3, 8, 8)]),
        ("mavg_nlc", "uniform", "moving_average", "per-tensor-affine", 8, "feature", "NLC", [(3, 7, 16), (3, 7, 16)]),
        ("aciqg_pt_s8", "uniform", "aciq:gaus", "per-tensor-symmetric", 8, "feature", "NCHW", [(4, 3, 12, 12)] * 2),
        ("aciqg_pt_a4", "uniform", "aciq:gaus", "per-tensor-affine", 4, "feature", "NCHW", [(4, 3, 12, 12)] * 2),
        ("aciqg_pc_w8", "uniform", "aciq:gaus", "per-channel-symmetric", 8, "weight", None, [(8, 5, 3, 3)]),
        ("aciql_pt_s8", "uniform", "aciq:laplace", "per-tensor-symmetric", 8, "feature", "NCHW", [(4, 3, 12, 12)] * 2),
        ("aciql_pc_w4", "uniform", "aciq:laplace", "per-channel-symmetric", 4, "weight", None, [(8, 5, 3, 3)]),
    ]
    for name, qtype, obs, scheme, bit, target, layout, shapes in specs:
        dist_mode = None
        if obs.startswith("aciq"):
            obs, dist_mode = obs.split(":")
        cfg = R.make_cfg(scheme, bit, target, obs, layout or "NCHW", qtype=qtype)
        if dist_mode:
            cfg.OBSERVER.ACIQ = R._CfgNode({"DISTRIBUTION": dist_mode})
        if target == "feature":
            cfg.QUANTIZER.PACT = R._CfgNode({"ALPHA_VALUE": 3})
            cfg.OBSERVER.MOVING_AVERAGE = R._CfgNode({"EMA_RATIO": 0.9})
        q = build_quantizer(cfg)
        q.set_backend(Backend.VIRTUAL)
        xs = []
        for i, shp in enumerate(shapes):
            x = torch.randn(shp, generator=g) * (1.0 + 0.5 * i)
            if "aff" in scheme and target == "feature" and qtype != "pact":
                x = torch.relu(x)
            xs.append(x)
            q.update_observer(x)
        with torch.no_grad():
            scale, zp = q.calc_qparams()
            q.enable_quant()
            y = q(xs[0])
            scale, zp = q._qparams_preprocess(xs[0]) if qtype in ("lsq", "lsq+", "pact") else (q.scale, q.zero_point)
        cases.append(name)
        for i, x in enumerate(xs):
            out[f"{name}_x{i}"] = x.numpy()
        out[name + "_nb"] = np.array(len(xs))
        out[name + "_scale"] = scale.detach().reshape(-1).numpy()
        out[name + "_zp"] = zp.detach().reshape(-1).numpy()
        out[name + "_y"] = y.detach().numpy()
        out[name + "_meta"] = np.array([q.qdesc.qmin, q.qdesc.qmax, q.qdesc.ch_axis, int(q.qdesc.is_perchannel), int(q.qdesc.is_symmetric), bit])
    out["cases"] = np.array(cases)
    # AdaRound (adaround.py): init_variables, eval (hard) and training (soft) forward, dL/dv by autograd
    ada = []
    for name, scheme, bit, shape in [("ada_pc_w4", "per-channel-symmetric", 4, (8, 5, 3, 3)),
                                     ("ada_pc_w8", "per-channel-symmetric", 8, (6, 16)),
                                     ("ada_pt_w4", "per-tensor-symmetric", 4, (8, 5, 3, 3)),
                                     ("ada_pt_a3", "per-tensor-affine", 3, (7, 9))]:
        cfg = R.make_cfg(scheme, bit, "weight", "minmax", "NCHW", qtype="adaround")
        q = build_quantizer(cfg)
        q.set_backend(Backend.VIRTUAL)
        w = torch.randn(shape, generator=g) * 0.2
        q.update_observer(w)
        q.calc_qparams()
        q.enable_quant()
        q.init_variables(w)
        v0 = q.v.detach().clone()
        v1 = (v0 + torch.randn(shape, generator=g) * 2.0).clone()
        q.v = torch.nn.Parameter(v1.clone())
        q.eval()
        with torch.no_grad():
            y_hard = q(w)
        q.train()
        y_soft = q(w)
        gy = torch.randn(shape, generator=g)
        (y_soft * gy).sum().backward()
        ada.append(name)
        out[name + "_w"] = w.numpy()
        out[name + "_v0"] = v0.numpy()
        out[name + "_v1"] = v1.numpy()
        out[name + "_scale"] = q.scale.detach().reshape(-1).numpy()
        out[name + "_zp"] = q.zero_point.detach().reshape(-1).numpy()
        out[name + "_yhard"] = y_hard.numpy()
        out[name + "_ysoft"] = y_soft.detach().numpy()
        out[name + "_gy"] = gy.numpy()
        out[name + "_gv"] = q.v.grad.numpy()
        out[name + "_meta"] = np.array([q.qdesc.qmin, q.qdesc.qmax, q.qdesc.ch_axis, int(q.qdesc.is_perchannel), int(q.qdesc.is_symmetric), bit])
    out["ada_cases"] = np.array(ada)
    save("next_rows", **out)


def gen_calibration():
    """SURVEY 8(f)#1: the reference's QuantModel + CalibrationRunner (tools/calibration.py) on a tiny CNN,
    CPU.  Records the weights, the calibration batches and every quantizer's resulting qparams."""
    import torch.nn as nn
    from sparsebit.quantization import QuantModel
    from sparsebit.quantization.quant_config import _C

    class Tiny(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1 = nn.Conv2d(3, 8, 3, padding=1)
            self.relu1 = nn.ReLU()
            self.conv2 = nn.Conv2d(8, 8, 3, stride=2)
            self.relu2 = nn.ReLU()
            self.fc = nn.Linear(8 * 3 * 3, 10)

        def forward(self, x):
            x = self.relu1(self.conv1(x))
            x = self.relu2(self.conv2(x))
            return self.fc(torch.flatten(x, 1))

    torch.manual_seed(7)
    net = Tiny().eval()
    g = torch.Generator().manual_seed(77)
    xs = [torch.randn(4, 3, 8, 8, generator=g) for _ in range(3)]
    out = {"nb": np.array(len(xs))}
    for k, v in net.state_dict().items():
        out["sd_" + k] = v.numpy()
    for i, x in enumerate(xs):
        out[f"x{i}"] = x.numpy()
    cases = []
    for name, wscheme, wbit, wobs, ascheme, abit, aobs in [
        ("mm8", "per-channel-symmetric", 8, "minmax", "per-tensor-affine", 8, "minmax"),
        ("pct", "per-channel-symmetric", 4, "minmax", "per-tensor-symmetric", 8, "percentile"),
        ("mse", "per-tensor-symmetric", 8, "mse", "per-tensor-affine", 4, "mse"),
        ("mavg", "per-channel-symmetric", 8, "minmax", "per-tensor-affine", 8, "moving_average"),
    ]:
        cfg = _C.clone()
        cfg.DEVICE = "cpu"
        cfg.W.QSCHEME, cfg.W.QUANTIZER.BIT, cfg.W.OBSERVER.TYPE = wscheme, wbit, wobs
        cfg.A.QSCHEME, cfg.A.QUANTIZER.BIT, cfg.A.OBSERVER.TYPE = ascheme, abit, aobs
        import copy

        qm = QuantModel(copy.deepcopy(net), cfg)
        qm.prepare_calibration()
        with torch.no_grad():
            for x in xs:
                qm(x)
        qm.calc_qparams()
        qm.set_quant(w_quant=True, a_quant=True)
        with torch.no_grad():
            y = qm(xs[0])
        cases.append(name)
        out[name + "_cfg"] = np.array([wscheme, str(wbit), wobs, ascheme, str(abit), aobs])
        for mod in ("conv1", "conv2", "fc"):
            m = getattr(qm.model, mod)
            out[f"{name}_{mod}_as"] = m.input_quantizer.scale.reshape(-1).numpy()
            out[f"{name}_{mod}_az"] = m.input_quantizer.zero_point.reshape(-1).numpy()
            out[f"{name}_{mod}_ws"] = m.weight_quantizer.scale.reshape(-1).numpy()
            out[f"{name}_{mod}_wz"] = m.weight_quantizer.zero_point.reshape(-1).numpy()
        for mod in ("relu1", "relu2"):  # fused away by DISABLE_UNNECESSARY_QUANT
            assert getattr(qm.model, mod).input_quantizer.fake_fused
        out[name + "_y"] = y.numpy()
    out["cases"] = np.array(cases)
    save("calibration", **out)


def gen_bwd():
    """STE backward known answers from the reference's own Python statement of it, ``MySTE.backward``
    (sparsebit/quantization/quantizers/quant_tensor.py:46-71; the production ``STE.backward`` is CUDA-only,
    :113-116).  ``MySTE.backward`` returns the ELEMENTWISE scale / zero-point gradient terms; they are stored
    as such (fp32) and reduced by the consumer.  ``ctx`` is a stand-in carrying what ``MySTE.forward`` saves
    (x, scale, zero_point.round(), qdesc)."""
    from sparsebit.quantization.quantizers.quant_tensor import MySTE

    g = torch.Generator().manual_seed(4242)
    out, cases = {}, []
    specs = [
        # name, shape, qscheme, bit, target, layout, scale multiplier (< 1 forces clipping)
        ("pt_sym8", (4, 3, 16, 16), "per-tensor-symmetric", 8, "feature", "NCHW", 0.5),
        ("pt_aff8", (4, 3, 16, 16), "per-tensor-affine", 8, "feature", "NCHW", 0.7),
        ("pt_aff4", (5, 37), "per-tensor-affine", 4, "feature", "NCHW", 1.0),
        ("pc_w_sym8", (6, 4, 3, 3), "per-channel-symmetric", 8, "weight", None, 0.6),
        ("pc_w_aff4", (7, 11), "per-channel-affine", 4, "weight", None, 0.8),
        ("pc_a_nchw_sym4", (3, 5, 7, 7), "per-channel-symmetric", 4, "feature", "NCHW", 0.5),
        ("pc_a_nlc_aff8", (3, 6, 8), "per-channel-affine", 8, "feature", "NLC", 0.7),
    ]
    for name, shape, scheme, bit, target, layout, mult in specs:
        cfg = R.make_cfg(scheme, bit, target, "minmax", layout or "NCHW")
        q = build_quantizer(cfg)
        q.set_backend(Backend.VIRTUAL)
        x = torch.randn(shape, generator=g) * 1.5
        if "aff" in name and target == "feature":
            x = torch.relu(x)
        q.update_observer(x)
        scale, zp = q.calc_qparams()
        scale = (scale * mult).clone()
        zp = zp.clone()
        if "aff" in name:
            zp = zp + 0.25  # learned (fractional) zero point: forward / backward use zero_point.round()
        flat = x.reshape(-1)
        s0 = float(scale.reshape(-1)[0])
        flat[0], flat[1], flat[2] = 0.5 * s0, 1.5 * s0, -2.5 * s0  # exact rounding ties
        gy = torch.randn(shape, generator=g)
        scale_p = scale.clone().requires_grad_(True)
        zp_r = zp.round().clone().requires_grad_(True)

        class Ctx:
            saved_tensors = (x, scale_p, zp_r)
            qdesc = q.qdesc

        with torch.no_grad():
            gin, gs_e, gz_e, _, _ = MySTE.backward(Ctx, gy)
        cases.append(name)
        out[name + "_x"] = x.numpy()
        out[name + "_gy"] = gy.numpy()
        out[name + "_scale"] = scale.reshape(-1).numpy()
        out[name + "_zp"] = zp.reshape(-1).numpy()
        out[name + "_gx"] = gin.numpy()
        out[name + "_gs_elem"] = gs_e.numpy()
        out[name + "_gz_elem"] = gz_e.numpy()
        out[name + "_meta"] = np.array([q.qdesc.qmin, q.qdesc.qmax, q.qdesc.ch_axis, int(q.qdesc.is_perchannel)])
    out["cases"] = np.array(cases)
    save("bwd", **out)


def gen_sparse_structured():
    """Structured (filter) pruning, sparse/sparsers/l1norm.py:27-40, and the SConv2d -> SBatchNorm2d mask hand-over
    (sparse/modules/conv.py:22-37, normalization.py:15-28) from the unmodified reference on CPU."""
    import torch.nn as nn
    from sparsebit.sparse.modules import SBatchNorm2d, SConv2d
    from sparsebit.sparse.sparsers import build_sparser

    g = torch.Generator().manual_seed(31337)
    out, cases = {}, []
    for name, shape, ratio in [("conv_r50", (16, 4, 3, 3), 0.5), ("conv_r30", (10, 3, 3, 3), 0.3), ("lin_r25", (12, 33), 0.25),
                               ("conv_r05", (8, 2, 1, 1), 0.05)]:
        cfg = R._CfgNode({"SPARSER": {"TYPE": "structed", "STRATEGY": "l1norm", "RATIO": ratio}})
        sp = build_sparser(cfg, opr=None)
        w = torch.randn(shape, generator=g)
        mask = sp.calc_mask(w)
        cases.append(name)
        out[name + "_w"] = w.numpy()
        out[name + "_mask"] = mask.numpy()
        out[name + "_ratio"] = np.array(ratio)
    out["cases"] = np.array(cases)
    # conv -> bn pair: the conv's filter mask is handed to the following SBatchNorm2d (sparse_model.py calc_params order)
    torch.manual_seed(5)
    conv, bn = nn.Conv2d(3, 8, 3, padding=1), nn.BatchNorm2d(8)
    with torch.no_grad():
        bn.weight.copy_(torch.randn(8, generator=g))
        bn.bias.copy_(torch.randn(8, generator=g))
        bn.running_mean.copy_(torch.randn(8, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(8, generator=g) + 0.5)
    cfg = R._CfgNode({"SPARSER": {"TYPE": "structed", "STRATEGY": "l1norm", "RATIO": 0.5}})
    sconv, sbn = SConv2d(conv, cfg), SBatchNorm2d(bn, cfg)
    sconv.build_sparser(cfg)
    sbn.build_sparser(cfg)
    pre = sconv.calc_mask()
    sbn.calc_mask(pre)
    x = torch.randn(2, 3, 6, 6, generator=g)
    sconv.eval(), sbn.eval()
    with torch.no_grad():
        y = sbn(sconv(x))
    for k, v in conv.state_dict().items():
        out["pair_conv_" + k] = v.numpy()
    for k, v in bn.state_dict().items():
        out["pair_bn_" + k] = v.numpy()
    out["pair_x"], out["pair_y"], out["pair_bn_mask"] = x.numpy(), y.numpy(), sbn.mask.numpy()
    save("sparse_structured", **out)


def _plant_grid_edges(x, s, zp, qmin, qmax, ch_axis=None):
    """Write rounding ties (k + 0.5)·s and values landing exactly on qmin / qmax (and half a step beyond them) at the head
    of every quantisation row of ``x`` (the whole tensor per tensor, each channel along ``ch_axis`` per channel)."""
    xn = x.numpy()
    rows = xn.reshape(1, -1) if ch_axis is None else np.moveaxis(xn, ch_axis, 0)
    s, zp = np.asarray(s, np.float32).reshape(-1), np.rint(np.asarray(zp, np.float32).reshape(-1))
    for c in range(rows.shape[0]):
        sc, z = s[min(c, s.size - 1)], zp[min(c, zp.size - 1)]
        units = [0.5, 1.5, -2.5, qmax - z - 0.5, qmin - z + 0.5, qmax - z, qmin - z, qmax - z + 0.5, qmin - z - 0.5]
        for i, u in enumerate(units):
            rows[c].flat[i] = np.float32(u) * sc


def gen_qat():
    """Train-mode gradients of the learnable quantizers (uniform, LSQ, LSQ+, PACT, DoReFa): calibrate, set the
    parameters, enable_quant, forward, ``(y * gy).sum().backward()``.  The production ``STE.backward`` is CUDA-only
    (quant_tensor.py:113-116), so ``STE`` is rebound in each quantizer module to a Function whose forward is the
    reference ``STE.forward`` (CPU fake-quant branch) and whose backward is the reference ``MySTE.backward``
    (quant_tensor.py:46-71), reduced to the parameter shapes.  Its ctx stand-in carries ``zero_point.round()`` as a
    tensor that still requires grad when the zero point does: ``MySTE.forward`` rounds under no-grad, which would drop
    the LSQ+ zero-point gradient.  MySTE differs from the per-channel CUDA kernel only in the zero-point rule (SURVEY
    Q4), which no case reaches: no per-channel zero point is learnable."""
    from sparsebit.quantization.quantizers import dorefa, lsq, lsq_plus, pact, uniform
    from sparsebit.quantization.quantizers import quant_tensor as qt

    class RefSTE(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, scale, zero_point, qdesc, backend):
            return qt.STE.forward(ctx, x, scale, zero_point, qdesc, backend)

        @staticmethod
        def backward(ctx, gout):
            x, scale, zero_point = ctx.saved_tensors
            need_s, need_z = ctx.needs_input_grad[1:3]

            class Ctx:
                saved_tensors = (x, scale.detach().requires_grad_(need_s), zero_point.detach().round().requires_grad_(need_z))
                qdesc = ctx.qdesc

            gx, gs, gz, _, _ = qt.MySTE.backward(Ctx, gout)
            return (gx, gs.sum_to_size(scale.shape) if need_s else None, gz.sum_to_size(zero_point.shape) if need_z else None,
                    None, None)

    for mod in (uniform, lsq, lsq_plus, pact, dorefa):
        mod.STE = RefSTE

    # the signed 8-bit PACT alpha whose bound alpha / scale lands just below 127.5 (rounds to qmax, not qmax + 1)
    al = np.linspace(1.0, 2.0, 4001, dtype=np.float32)
    sc = (al * np.float32(2)) / np.float32(255)
    alpha_qmax = float(al[np.rint(al / sc) == 127][0])

    g = torch.Generator().manual_seed(515)
    out, cases = {}, []
    specs = [
        # name, qtype, scheme, bit, target, layout, shape, x multiplier, parameter setup
        ("uni_pt_s8", "uniform", "per-tensor-symmetric", 8, "feature", "NCHW", (2, 3, 5, 5), 1.5, None),
        ("uni_pt_a8_nlc", "uniform", "per-tensor-affine", 8, "feature", "NLC", (2, 6, 12), 1.5, None),
        ("uni_pc_w4", "uniform", "per-channel-symmetric", 4, "weight", None, (6, 4, 3, 3), 0.3, None),
        ("lsq_pt_s4", "lsq", "per-tensor-symmetric", 4, "feature", "NCHW", (2, 3, 5, 5), 1.5, None),
        ("lsq_pc_conv4", "lsq", "per-channel-symmetric", 4, "weight", None, (16, 8, 3, 3), 0.3, None),
        ("lsq_pc_lin8", "lsq", "per-channel-symmetric", 8, "weight", None, (24, 40), 0.3, None),
        ("lsq_pc_neg4", "lsq", "per-channel-symmetric", 4, "weight", None, (6, 4, 3, 3), 0.3, "negate_scale"),
        ("lsqp_pt_a8_half", "lsq+", "per-tensor-affine", 8, "feature", "NCHW", (2, 3, 5, 5), 1.5, "zp_half"),
        ("lsqp_pt_a8_qmin", "lsq+", "per-tensor-affine", 8, "feature", "NCHW", (2, 3, 5, 5), 1.5, "zp_qmin"),
        ("lsqp_pt_a8_above", "lsq+", "per-tensor-affine", 8, "feature", "NCHW", (2, 3, 5, 5), 1.5, "zp_above"),
        ("lsqp_pc_w4", "lsq+", "per-channel-symmetric", 4, "weight", None, (6, 4, 3, 3), 0.3, None),
        ("pact_s8_a15", "pact", "per-tensor-symmetric", 8, "feature", "NCHW", (4, 3, 16, 16), 2.0, 1.5),
        ("pact_s4_a30", "pact", "per-tensor-symmetric", 4, "feature", "NCHW", (2, 3, 5, 5), 2.5, 3.0),
        ("pact_s8_qmax", "pact", "per-tensor-symmetric", 8, "feature", "NCHW", (2, 3, 5, 5), 1.5, alpha_qmax),
        ("pact_u8", "pact", "per-tensor-affine", 8, "feature", "NCHW", (2, 3, 5, 5), 1.5, 1.5),
        ("pact_u4", "pact", "per-tensor-affine", 4, "feature", "NCHW", (2, 3, 5, 5), 2.5, 3.0),
        ("dorefa_w4", "dorefa", "per-tensor-symmetric", 4, "weight", None, (6, 4, 3, 3), 0.6, None),
    ]
    for name, qtype, scheme, bit, target, layout, shape, mult, setup in specs:
        cfg = R.make_cfg(scheme, bit, target, "minmax", layout or "NCHW", qtype=qtype)
        if qtype == "pact":
            cfg.QUANTIZER.PACT = R._CfgNode({"ALPHA_VALUE": setup})
        q = build_quantizer(cfg)
        q.set_backend(Backend.VIRTUAL)
        if name == "pact_s8_a15":  # the inputs of the worked example in SURVEY Q19: alpha.grad = 45.153
            gp = torch.Generator().manual_seed(0)
            x = torch.randn(shape, generator=gp) * mult
            gy = torch.randn(shape, generator=gp)
        else:
            x = torch.randn(shape, generator=g) * mult
            gy = torch.randn(shape, generator=g)
        q.update_observer(x)
        q.calc_qparams()
        with torch.no_grad():
            if setup == "negate_scale":
                q.scale[::3] *= -1
            elif setup in ("zp_half", "zp_qmin", "zp_above"):
                z = {"zp_half": float(torch.round(q.zero_point).reshape(-1)[0]) + 0.5, "zp_qmin": float(q.qdesc.qmin),
                     "zp_above": float(q.qdesc.qmax) + 9.25}[setup]
                q.zero_point.fill_(z)
            s_used, z_used = q._qparams_preprocess(x)
            if qtype == "dorefa":  # ties of the normalised tensor: x = atanh(u * s * max|tanh x|), the maximum kept
                t_ = x.tanh()
                m = t_.abs().max()
                u = torch.tensor([0.5, 1.5, -2.5, 6.5, -6.5, 7.0]) * q.scale.reshape(-1)[0] * m
                keep = int(t_.abs().reshape(-1).argmax())
                pos = [i for i in range(8) if i != keep][: u.numel()]
                x.reshape(-1)[pos] = torch.atanh(u)
            elif name != "pact_s8_a15":
                ch = q.qdesc.ch_axis if q.qdesc.is_perchannel else None
                _plant_grid_edges(x, s_used.detach(), z_used.detach(), q.qdesc.qmin, q.qdesc.qmax, ch)
                if qtype == "pact":  # the clamp bounds themselves and one ulp either side
                    a = np.float32(setup)
                    lo = -a if q.qdesc.qmin < 0 else np.float32(0)
                    bounds = [a, np.nextafter(a, np.float32(0)), np.nextafter(a, np.float32(9)), lo,
                              np.nextafter(lo, np.float32(-9)), np.nextafter(lo, np.float32(9))]
                    x.reshape(-1)[9:9 + len(bounds)] = torch.tensor(bounds)
        q.enable_quant()
        xr = x.clone().requires_grad_(True)
        y = q(xr)
        (y * gy).sum().backward()
        cases.append(name)
        qd = q.qdesc
        out[name + "_cfg"] = np.array([qtype, scheme, target, layout or ""])
        out[name + "_meta"] = np.array([qd.qmin, qd.qmax, qd.ch_axis, int(qd.is_perchannel), int(qd.is_symmetric), bit])
        out[name + "_x"], out[name + "_gy"] = x.numpy(), gy.numpy()
        out[name + "_y"], out[name + "_gx"] = y.detach().numpy(), xr.grad.numpy()
        if qtype == "pact":
            out[name + "_alpha"] = q.alpha.detach().numpy()
            out[name + "_galpha"] = q.alpha.grad.numpy()
            continue
        out[name + "_scale"] = q.scale.detach().reshape(-1).numpy()
        out[name + "_zp"] = q.zero_point.detach().reshape(-1).numpy()
        if q.scale.grad is not None:
            out[name + "_gscale"] = q.scale.grad.reshape(-1).numpy()
        if isinstance(q.zero_point, torch.nn.Parameter) and q.zero_point.grad is not None:
            out[name + "_gzp"] = q.zero_point.grad.reshape(-1).numpy()
    out["cases"] = np.array(cases)
    save("qat", **out)


GENERATORS = {"qdq": gen_qdq, "observers": gen_observers, "sparse": gen_sparse, "gptq": gen_gptq,
              "next_rows": gen_next_rows, "calibration": gen_calibration, "bwd": gen_bwd,
              "sparse_structured": gen_sparse_structured, "qat": gen_qat}

if __name__ == "__main__":
    torch.set_num_threads(4)
    for which in sys.argv[1:] or list(GENERATORS):  # e.g. `make_golden.py bwd` regenerates one fixture
        GENERATORS[which]()
