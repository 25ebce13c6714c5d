"""GPU parity for the streaming, device-resident CalibrationRunner (SURVEY 8f #1) against the
reference's QuantModel + CalibrationRunner run on CPU (tests/golden/make_golden.py::gen_calibration)."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from gpu_util import bits_equal, dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.modules import QConv2d, QLinear, QReLU
from sparsebit_b200.quantization.tools import CalibrationRunner, trace_quant_model

pytestmark = pytest.mark.gpu


class Tiny(nn.Module):
    """What the reference's QuantModel turns the golden generator's CNN into: QConv2d / QReLU / QLinear with
    the ReLU input quantizers fused away (SCHEDULE.DISABLE_UNNECESSARY_QUANT)."""

    def __init__(self, g, case, wtype="uniform"):
        super().__init__()
        wscheme, wbit, wobs, ascheme, abit, aobs = (str(v) for v in g[case + "_cfg"])
        conv1, conv2, fc = nn.Conv2d(3, 8, 3, padding=1), nn.Conv2d(8, 8, 3, stride=2), nn.Linear(72, 10)
        with torch.no_grad():
            for name, mod in (("conv1", conv1), ("conv2", conv2), ("fc", fc)):
                mod.weight.copy_(torch.from_numpy(g[f"sd_{name}.weight"]))
                mod.bias.copy_(torch.from_numpy(g[f"sd_{name}.bias"]))

        def a_cfg(disable=False):
            return sbcfg.quantizer_config(ascheme, int(abit), "feature", aobs, disable=disable)

        def w_cfg():
            return sbcfg.quantizer_config(wscheme, int(wbit), "weight", wobs, qtype=wtype)

        self.conv1 = QConv2d(conv1).build_quantizer(a_cfg(), w_cfg())
        self.relu1 = QReLU().build_quantizer(a_cfg(disable=True))
        self.conv2 = QConv2d(conv2).build_quantizer(a_cfg(), w_cfg())
        self.relu2 = QReLU().build_quantizer(a_cfg(disable=True))
        self.fc = QLinear(fc).build_quantizer(a_cfg(), w_cfg())

    def forward(self, x):
        x = self.relu1(self.conv1(x))
        x = self.relu2(self.conv2(x))
        return self.fc(torch.flatten(x, 1))


def _calibrate(g, case, streaming=True, asym=False, **kw):
    model = trace_quant_model(Tiny(g, case, **kw).to(dev()))
    runner = CalibrationRunner(model, streaming=streaming)
    runner.adaround_kwargs = dict(max_steps=150, batch_size=8, print_freq=0)
    runner.prepare_calibration()
    with torch.no_grad():
        for i in range(int(g["nb"])):
            model(t(g[f"x{i}"]))
    runner.layerwise_calibration(dev(), asym=asym, w_quant=asym, a_quant=asym)
    return model


def _qparams(model):
    out = {}
    for name in ("conv1", "conv2", "fc"):
        m = getattr(model, name)
        out[name] = tuple(v.reshape(-1).cpu().numpy() for v in (m.input_quantizer.scale, m.input_quantizer.zero_point,
                                                                m.weight_quantizer.scale, m.weight_quantizer.zero_point))
    return out


def test_streaming_runner_matches_reference_quantmodel(golden):
    g = golden("calibration")
    for case in g["cases"]:
        case = str(case)
        model = _calibrate(g, case)
        qp = _qparams(model)
        for name in ("conv1", "conv2", "fc"):
            a_s, a_z, w_s, w_z = qp[name]
            # weights, and the first layer's input (the raw calibration batches): same data -> bit-exact
            assert bits_equal(w_s, g[f"{case}_{name}_ws"]) and bits_equal(w_z, g[f"{case}_{name}_wz"]), (case, name)
            if name == "conv1":
                assert bits_equal(a_s, g[f"{case}_{name}_as"]) and bits_equal(a_z, g[f"{case}_{name}_az"]), (case, name)
            else:
                # inputs produced by cuDNN / cuBLAS instead of the CPU conv: float tolerance; the MSE
                # observer's argmin over 80 candidates may move by one 1 % step on such perturbations
                tol = 2.5e-2 if case == "mse" else 1e-4
                np.testing.assert_allclose(a_s, g[f"{case}_{name}_as"], rtol=tol, err_msg=f"{case} {name}")
                assert np.max(np.abs(a_z - g[f"{case}_{name}_az"])) <= (1 if case == "mse" else 0), (case, name)
        # nothing is left cached on the device, hooks are gone, relu quantizers stay fused
        for m in model.modules():
            if getattr(m, "input_quantizer", None) is not None:
                assert len(m.input_quantizer.observer.data_cache) == 0
                assert len(m._forward_pre_hooks) == 0
        assert model.relu1.input_quantizer.fake_fused and float(model.relu1.input_quantizer.scale) == 1.0
        # end to end: quantized forward of the calibrated model
        for m in (model.conv1, model.relu1, model.conv2, model.relu2, model.fc):
            m.set_quant(w_quant=True, a_quant=True)
        with torch.no_grad():
            y = model(t(g["x0"])).cpu().numpy()
        gy = g[case + "_y"]
        assert np.mean(np.abs(y - gy)) < 0.03 * np.mean(np.abs(gy)), case


def test_layerwise_replay_equals_streaming(golden):
    """The device-resident replay (used for asym / AdaRound) and the streaming path see the same data."""
    g = golden("calibration")
    for case in ("mm8", "pct"):
        base = _qparams(_calibrate(g, case, streaming=True))
        for streaming, asym in ((False, False), (True, True), (False, True)):
            other = _qparams(_calibrate(g, case, streaming=streaming, asym=asym))
            for name in base:
                for a, b in zip(base[name], other[name]):
                    assert bits_equal(a, b), (case, name, streaming, asym)


def test_adaround_layerwise_reconstruction(golden):
    g = golden("calibration")
    model = _calibrate(g, "pct", wtype="adaround", asym=True)
    for name in ("conv1", "conv2", "fc"):
        wq = getattr(model, name).weight_quantizer
        assert wq.v.shape == getattr(model, name).weight.shape and not wq.training
        assert torch.isfinite(wq.v).all()
    for m in (model.conv1, model.relu1, model.conv2, model.relu2, model.fc):
        m.set_quant(w_quant=True, a_quant=False)
    with torch.no_grad():
        y = model(t(g["x0"]))
        w = model.fc.weight
        wq = model.fc.weight_quantizer
        dq = wq(w)
        # eval branch: every weight sits on the 4-bit grid, one of the two neighbours of w / scale
        steps = dq / wq.scale
        assert torch.allclose(steps, steps.round(), atol=1e-4)
        assert ((steps - w / wq.scale).abs() <= 1.0 + 1e-4).all()
    assert torch.isfinite(y).all()
