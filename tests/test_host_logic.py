"""CPU: host-side logic of the plugin mirror -- registries, descriptors, qparams math, the KL
entropy search, GPTQ packing -- against the oracle and the reference's golden vectors."""
import os

import numpy as np
import pytest
import torch

from oracle import gptq as ogptq
from oracle import observers as oobs
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.gptq.quant_linear import QuantLinear, find_params_int4
from sparsebit_b200.quantization import OBSERVERS_MAP, QUANTIZERS_MAP, build_observer, build_quantizer
from sparsebit_b200.quantization.common import Backend, get_backend, get_qscheme
from sparsebit_b200.quantization.observers.kl_histogram import entropy_threshold
from sparsebit_b200.quantization.quant_descriptor import QuantDescriptor
from sparsebit_b200.sparse import SPARSERS_MAP, build_sparser


def test_registries_hold_reference_type_names():
    assert "uniform" in QUANTIZERS_MAP
    assert {"minmax", "mse", "percentile", "kl_histogram"} <= set(OBSERVERS_MAP)
    assert "l1norm" in SPARSERS_MAP
    with pytest.raises(AssertionError):  # reference asserts before lower-casing (Q18)
        build_quantizer(sbcfg.quantizer_config("per-tensor-affine", 8, "feature", qtype="Uniform"))
    with pytest.raises(TypeError):
        get_qscheme("per-tensor")
    assert get_backend("tensorrt") is Backend.TENSORRT


@pytest.mark.parametrize(
    "scheme,bit,target,layout,exp",
    [
        ("per-tensor-symmetric", 8, "feature", "NCHW", (-128, 127, 1, 0, False, True)),
        ("per-tensor-affine", 4, "feature", "NLC", (0, 15, 2, 0, False, False)),
        ("per-channel-symmetric", 4, "weight", None, (-8, 7, 0, None, True, True)),
        ("per-channel-affine", 8, "weight", None, (0, 255, 0, None, True, False)),
    ],
)
def test_quant_descriptor(scheme, bit, target, layout, exp):
    d = QuantDescriptor(sbcfg.quantizer_config(scheme, bit, target, layout=layout or "NCHW"))
    assert (d.qmin, d.qmax, d.ch_axis, d.bs_axis, d.is_perchannel, d.is_symmetric) == exp
    assert d.qrange == (d.qmin, d.qmax)
    d.set_bit(2)
    assert d.qrange == ((-2, 1) if d.is_symmetric else (0, 3))


@pytest.mark.parametrize("sym", [True, False])
def test_calc_qparams_with_minmax_matches_oracle(sym):
    scheme = "per-channel-symmetric" if sym else "per-channel-affine"
    cfg = sbcfg.quantizer_config(scheme, 8, "weight")
    obs = build_observer(cfg, QuantDescriptor(cfg))
    g = torch.Generator().manual_seed(0)
    mn = -torch.rand(64, generator=g) * 3
    mx = torch.rand(64, generator=g) * 5
    mn[:4] = 0.3  # positive minimum -> clamped to 0
    mx[4:8] = -0.2
    mn[8], mx[8] = 0.0, 0.0  # degenerate -> scale floor 1e-6
    s, z = obs.calc_qparams_with_minmax(mn, mx)
    so, zo = oobs.calc_qparams_with_minmax(mn.numpy(), mx.numpy(), *obs.qdesc.qrange, sym)
    assert np.array_equal(s.numpy(), so)
    assert np.array_equal(z.numpy() + 0.0, zo + 0.0)


@pytest.mark.parametrize("bit", [8, 4])
def test_entropy_threshold_matches_reference_restatement(bit):
    rng = np.random.default_rng(bit)
    for trial in range(3):
        x = (rng.standard_normal(20000) * (1 + trial)).astype(np.float32)
        if trial == 2:
            x = np.abs(x)
        am = np.abs(x).max()
        hist = oobs.histc(x, 2048, -am, am).astype(np.float32)
        a = oobs.calibrate_entropy(hist, 1.0, 2048, 2**bit - 1)
        b = entropy_threshold(hist, 1.0, 2048, 2**bit - 1)
        assert a == b
    # the documented degenerate behaviour (SURVEY Q6): slot 1025 - 2^bit wins on ordinary data
    assert b == 1025 - 2**bit


def test_gptq_pack_and_find_params_match_reference(golden):
    g = golden("gptq")
    for name in g["cases"]:
        gs = int(g[name + "_gs"])
        w = torch.from_numpy(g[name + "_wdq"])
        n, k = w.shape
        scale, zero = find_params_int4(w, gs)
        np.testing.assert_array_equal(zero.reshape(n, -1).numpy(), g[name + "_zero_int"])
        lin = torch.nn.Linear(k, n)
        lin.weight.data = w
        lin.bias.data = torch.from_numpy(g[name + "_bias"])
        ql = QuantLinear(k, n, bit=4, groupsize=gs)
        ql.pack(lin, scale, zero)
        np.testing.assert_array_equal(ql.qweight.numpy(), g[name + "_qweight"])
        np.testing.assert_allclose(ql.scales.reshape(n, -1).numpy(), g[name + "_scales"], rtol=1e-6)
        np.testing.assert_allclose(ql.zeros.reshape(n, -1).numpy(), g[name + "_zeros"], rtol=1e-6, atol=1e-9)
        # and the oracle's packer agrees with both
        qw2, _, _ = ogptq.pack_int4(g[name + "_wdq"], scale.reshape(n, -1).numpy(), zero.reshape(n, -1).numpy())
        np.testing.assert_array_equal(qw2, g[name + "_qweight"])


def test_sparser_builds_and_ratio_zero_is_ones():
    sp = build_sparser(sbcfg.sparser_config(0.0), opr=None)
    w = torch.randn(3, 4)
    assert torch.equal(sp.calc_mask(w), torch.ones_like(w))
    assert repr(sp) == "unstructed, l1norm, 0.0"
    sp.set_ratio(0.5)
    assert sp.ratio == 0.5


def test_quantizer_state_contract():
    q = build_quantizer(sbcfg.quantizer_config("per-channel-symmetric", 8, "weight"))
    assert set(dict(q.named_buffers())) >= {"scale", "zero_point", "observer.min_val", "observer.max_val"}
    assert not q.is_enable
    q.enable_quant()
    assert q.is_enable
    q.set_fake_fused()
    assert not q.is_enable
    x = torch.randn(4, 4)
    assert q(x) is x  # disabled quantizer is the identity (base.py:55-64)
    q.set_backend(Backend.VIRTUAL)
    assert q.observer.backend is Backend.VIRTUAL
    q.dims = 4
    assert q._broadcast_qparams(torch.ones(6)).shape == (6, 1, 1, 1)


# ---------------------------------------------------------------- CalibrationRunner host logic (no kernels)
class _StubCache(list):
    def reset(self):
        self.clear()


class _StubObserver:
    def __init__(self):
        self.data_cache = _StubCache()


class _StubQuantizer:
    TYPE = "uniform"

    def __init__(self, fused=False):
        self.fake_fused = fused
        self.seen, self.calcs = [], 0
        self.observer = _StubObserver()

    def update_observer(self, x):
        self.seen.append(tuple(x.shape))

    def calc_qparams(self):  # a foreign quantizer without calc_qparams_steps: the runner calls this as one step
        self.calcs += 1


def _stub_net():
    import torch

    class Opr(torch.nn.Module):
        def __init__(self, has_weight, fused=False):
            super().__init__()
            self.input_quantizer = _StubQuantizer(fused)
            self.weight_quantizer = _StubQuantizer() if has_weight else None
            self.weight = torch.nn.Parameter(torch.ones(2, 2)) if has_weight else None
            self.flags = None

        def set_quant(self, w_quant=False, a_quant=False):
            self.flags = (w_quant, a_quant)

        def forward(self, x):
            return x * 2 if self.weight is not None else x + 1

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.a, self.b, self.c = Opr(True), Opr(False, fused=True), Opr(True)

        def forward(self, x):
            h = self.a(x)
            return self.c(self.b(h) + h)

    return Net()


def test_calibration_runner_streaming_and_replay_feed_the_same_batches():
    import torch

    from sparsebit_b200.quantization.tools import CalibrationRunner, trace_quant_model

    batches = [torch.zeros(3, 4), torch.zeros(5, 4)]
    for streaming, asym in ((True, False), (False, False), (True, True)):
        net = trace_quant_model(_stub_net())
        assert [n.op for n in net.graph.nodes].count("call_module") == 3  # quant operators stay leaves
        runner = CalibrationRunner(net, streaming=streaming)
        runner.prepare_calibration()
        for x in batches:
            # the reference's QuantModel.forward calls the graph module's .forward directly (quant_model.py:206-207),
            # which bypasses hooks on the graph module itself: the inputs must still be captured for the replay
            net.forward(x) if asym else net(x)
        runner.layerwise_calibration(None, asym=asym, w_quant=asym, a_quant=asym)
        assert all(len(m._forward_pre_hooks) == 0 for m in net.modules())
        # live input quantizers see every batch once per pass (a replay after streaming feeds them again,
        # after resetting the observers' caches)
        expect = [(3, 4), (5, 4)] * (2 if (streaming and asym) else 1)
        assert net.a.input_quantizer.seen == expect and net.c.input_quantizer.seen == expect
        assert net.b.input_quantizer.seen == [] and net.b.input_quantizer.calcs == 0  # fake-fused: untouched
        assert net.a.input_quantizer.calcs == 1 and net.c.weight_quantizer.calcs == 1
        assert net.a.weight_quantizer.seen == [(2, 2)]
        if asym or not streaming:
            assert net.a.flags == (False, False)  # quant switched back off after each replayed node


def test_sparse_operator_with_a_built_sparser_is_not_a_cyclic_module():
    """SparseOpr.build_sparser hands the operator to its sparser (sparse/modules/base.py:23-24 passes a repr
    string): the sparser must not register it back as a submodule."""
    from sparsebit_b200.sparse.modules import SConv2d, SLinear

    for m in (SLinear(torch.nn.Linear(4, 3)), SConv2d(torch.nn.Conv2d(2, 3, 3))):
        m.build_sparser(sbcfg.sparser_config(0.5))
        assert m.sparser.opr is m
        m.eval()
        m.to("cpu")
        assert set(m.state_dict()) >= {"weight", "w_mask"}
        assert sum(1 for _ in m.modules()) == 2  # the operator and its sparser, nothing recursive


def test_data_cache_reset_also_drops_the_owners_streaming_state():
    """The reference idiom ``observer.data_cache.reset()`` (tools/calibration.py:113) must not leave a running
    min/max, per-sample extrema or element counts behind (a replay would otherwise see every batch twice)."""
    from sparsebit_b200.quantization.observers import build_observer
    from sparsebit_b200.quantization.quant_descriptor import QuantDescriptor

    cfg = sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature", observer="aciq")
    obs = build_observer(cfg, QuantDescriptor(cfg))
    obs._mm_state, obs._numel = torch.zeros(2, dtype=torch.int32), 1234
    obs.data_cache._batches, obs.data_cache._batch_size = 3, 12
    obs.data_cache.reset()
    assert obs._mm_state is None and obs._numel == 0 and len(obs.data_cache) == 0
    cfg = sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature", observer="moving_average")
    obs = build_observer(cfg, QuantDescriptor(cfg))
    obs._per_sample = [torch.zeros(2, 3)]
    obs.data_cache.reset()
    assert obs._per_sample == []
    # release() only drops the retained batches
    obs._mm_state = torch.zeros(2, dtype=torch.int32)
    obs.data_cache._tensors, obs.data_cache._batches = [torch.zeros(1)], 1
    obs.data_cache.release()
    assert obs._mm_state is not None and len(obs.data_cache) == 0


def test_quantlinear_pack_layouts_match_reference(golden):
    """Host-side QuantLinear.pack (vectorised) vs the reference's packed words, all three bit widths."""
    import torch

    from sparsebit_b200.gptq.quant_linear import QuantLinear, pack_rows

    for fixture in ("gptq", "gptq_lowbit"):
        g = golden(fixture)
        for name in g["cases"]:
            bit, gs = (4, int(g[name + "_gs"])) if fixture == "gptq" else (int(v) for v in g[name + "_meta"])
            wdq = torch.from_numpy(g[name + "_wdq"])
            n, k = wdq.shape
            lin = torch.nn.Linear(k, n)
            lin.weight.data, lin.bias.data = wdq, torch.from_numpy(g[name + "_bias"])
            s = torch.from_numpy(g[name + "_scales"])
            zi = torch.from_numpy(g[name + "_zero_int"])
            shape = (n, s.shape[1], 1) if gs != -1 else (n, 1)
            ql = QuantLinear(k, n, bit=bit, groupsize=gs)
            assert ql.qweight.shape == (pack_rows(k, bit), n)
            ql.pack(lin, s.reshape(shape), zi.reshape(shape))
            assert torch.equal(ql.qweight, torch.from_numpy(g[name + "_qweight"])), (name, bit)
            assert torch.equal(ql.zeros.reshape(n, -1), torch.from_numpy(g[name + "_zeros"])), name


@pytest.mark.skipif(not os.path.isdir("/root/reference/sparsebit"), reason="needs the reference checkout (build container only)")
def test_install_rebinds_reference_calibration_runner():
    """INTEGRATION.md section 1: with the unmodified reference importable, install() puts the streaming runner
    under QuantModel.prepare_calibration and the device observers under the reference's registry; without a
    GPU the first observer update fails loudly instead of falling back to a CPU path."""
    import subprocess
    import sys
    import textwrap

    code = textwrap.dedent("""
        import sys
        sys.path.insert(0, "tests/golden")
        import _ref_import as R
        R.install_shims()
        import torch, torch.nn as nn
        import sparsebit_b200
        sparsebit_b200.install()
        from sparsebit.quantization import QuantModel
        from sparsebit.quantization.quant_config import _C

        class Tiny(nn.Module):
            def __init__(self):
                super().__init__()
                self.conv1 = nn.Conv2d(3, 8, 3, padding=1); self.relu1 = nn.ReLU(); self.fc = nn.Linear(512, 10)
            def forward(self, x):
                return self.fc(torch.flatten(self.relu1(self.conv1(x)), 1))

        cfg = _C.clone(); cfg.DEVICE = "cpu"
        cfg.W.QSCHEME = "per-channel-symmetric"; cfg.W.QUANTIZER.BIT = 8
        cfg.A.QSCHEME = "per-tensor-affine"; cfg.A.QUANTIZER.BIT = 8
        qm = QuantModel(Tiny().eval(), cfg)
        qm.prepare_calibration()
        assert type(qm.calibration_runner).__module__ == "sparsebit_b200.quantization.tools.calibration"
        assert type(qm.model.conv1.input_quantizer.observer).__module__.startswith("sparsebit_b200.")
        # observer feed on every quant operator; the graph input is captured at its first consumer (conv1)
        assert [len(m._forward_pre_hooks) for m in (qm.model, qm.model.conv1, qm.model.relu1, qm.model.fc)] == [0, 2, 1, 1]
        try:
            qm(torch.randn(2, 3, 8, 8))
        except RuntimeError as e:
            assert "no CPU fallback" in str(e), e
            print("LOUD")
        else:
            print("CUDA" if torch.cuda.is_available() else "SILENT")
    """)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip().splitlines()[-1] in ("LOUD", "CUDA")


def test_kl_entropy_screen_equals_index_exact_search():
    """entropy_threshold's vectorised screen must return exactly what the index-exact restatement of
    calibrate_entropy (kl_histogram.py:54-94) returns -- including histograms where some candidate's
    divergence is ~0 and argmin does NOT land on the never-written slot."""
    from sparsebit_b200.quantization.observers import kl_histogram as K

    rng = np.random.default_rng(5)
    hists = []
    for trial in range(3):
        x = rng.standard_normal(60_000) * (1 + trial)
        x = np.abs(x) if trial == 1 else x
        am = np.abs(x).max()
        hists.append(np.histogram(x, bins=2048, range=(-am, am))[0].astype(np.float32))
    x = np.round(rng.standard_normal(5000) * 2)  # sparse histogram: exercises the exact fallback
    hists.append(np.histogram(x, bins=2048, range=(-np.abs(x).max(), np.abs(x).max()))[0].astype(np.float32))
    hists += [np.zeros(2048, np.float32), np.eye(1, 2048, 1024, dtype=np.float32)[0] * 1000, np.ones(2048, np.float32)]
    landed_elsewhere = 0
    for h in hists:
        for dst in (255, 15):
            exact = K._entropy_threshold_exact(h, 1.0, 2048, dst)
            assert K.entropy_threshold(h, 1.0, 2048, dst) == exact
            landed_elsewhere += exact not in (769.0, 1009.0)
    assert landed_elsewhere >= 3  # the fallback path was really taken
    cand, div = K._divergences_fp64(hists[0], 2048, 255)
    assert len(cand) == 897 and np.all(div > 1e-4)


def test_tcgen05_numeric_scheme_meets_the_reference_tolerance():
    """CPU emulation of the arithmetic the per-group wgmma GPTQ kernel performs (gptq_tc.cu header): activations scaled
    by a per-row power of two and split into fp16 hi + lo, exact int4 (minus integer zero) fp16 operands, fp32
    accumulation per 128-K group, fp32 fold `acc += scale * partial`, final `out += rowscale * acc`.  The
    scheme -- not a particular GPU -- must stay inside the reference's rtol = atol = 1e-5 (test_cuda_kernel.py:47)
    against the fp64 oracle, including outlier activations and the fp16-exact single-pass mode."""
    rng = np.random.default_rng(3)
    k, n, gs = 1024, 48, 128
    for case in ("normal", "outliers", "fp16_acts", "tiny_scales"):
        w = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
        if case == "tiny_scales":
            w *= 1e-3
        scale, zero = ogptq.find_params_int4(w, gs)
        wq = ogptq.quantize_weight(w, scale, zero, gs)
        qw, scales, zeros = ogptq.pack_int4(wq, scale, zero)
        x = rng.standard_normal((9, k)).astype(np.float32)
        if case == "outliers":
            x[:, ::97] *= 300.0
            x[3] *= 1e-4
        if case == "fp16_acts":
            x = x.astype(np.float16).astype(np.float32)
        bias = (rng.standard_normal(n) * 0.1).astype(np.float32)
        exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (9, n)), scales, zeros, gs)

        q = ogptq.unpack_int4(qw, k).astype(np.float32)                      # [K, N], exact in fp16
        zint = np.rint(zeros / scales).astype(np.float32)                     # integer zero points [N, G]
        assert np.all(np.abs(zeros - zint * scales) <= np.abs(zeros) * 2.0**-20 + 1e-30)
        amax = np.abs(x).max(axis=1)
        e = np.where(amax > 0, np.floor(np.log2(np.maximum(amax, 1e-38))) - 14, 0).astype(np.int32)
        xs = np.ldexp(x, -e[:, None]).astype(np.float32)                      # row max in [2^14, 2^15)
        hi = xs.astype(np.float16)
        lo = (xs - hi.astype(np.float32)).astype(np.float16)
        if case == "fp16_acts":
            assert not lo.any()                                               # the kernel skips the second MMA pass
        acc = np.zeros((9, n), np.float32)
        for g in range(k // gs):
            sl = slice(g * gs, (g + 1) * gs)
            b = (q[sl] - zint[:, g][None, :]).astype(np.float16)              # operand of the MMA, exact
            assert np.array_equal(b.astype(np.float32), q[sl] - zint[:, g][None, :])
            # fp16 x fp16 products are exact in fp32; the accumulation order of the tensor core is unspecified:
            # emulate it with an fp32 running sum over k (the least favourable ordering a GPU could use)
            part = np.zeros((9, n), np.float32)
            for kk in range(gs):
                part += hi[:, sl][:, kk:kk + 1].astype(np.float32) * b[kk][None, :].astype(np.float32)
                part += lo[:, sl][:, kk:kk + 1].astype(np.float32) * b[kk][None, :].astype(np.float32)
            acc = (acc + scales[:, g][None, :] * part).astype(np.float32)
        got = (np.broadcast_to(bias, (9, n)) + np.ldexp(acc, e[:, None])).astype(np.float32)
        np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-5, err_msg=case)


def test_qdq_onnx_export_emits_quantize_dequantize_linear(monkeypatch):
    """QDQ-ONNX export (quant_model.py:217-260 -> quant_tensor.py:220-249): with ``export_onnx`` set, Quantizer.forward
    must stay on the stock ATen fake-quantize ops so that the exporter emits QuantizeLinear / DequantizeLinear -- the
    custom kernels are not involved.  (The ``onnx`` Python package is absent in this image; the TorchScript exporter
    only needs it for a post-processing hook that is irrelevant here, so the hook is bypassed and the serialized graph
    is inspected as bytes.)"""
    import io
    import warnings

    from torch.onnx._internal.torchscript_exporter import onnx_proto_utils

    monkeypatch.setattr(onnx_proto_utils, "_add_onnxscript_fn", lambda proto, custom_opsets: proto)

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(8, 4)
            self.aq = build_quantizer(sbcfg.quantizer_config("per-tensor-affine", 8, "feature"))
            self.wq = build_quantizer(sbcfg.quantizer_config("per-channel-symmetric", 8, "weight"))

        def forward(self, x):
            return torch.nn.functional.linear(self.aq(x), self.wq(self.lin.weight), self.lin.bias)

    m = M().cpu().eval()
    for q, s, z in ((m.aq, torch.tensor([0.05]), torch.tensor([3.0])), (m.wq, torch.rand(4, 1) * 0.01 + 0.01, torch.zeros(4, 1))):
        q.scale, q.zero_point = s, z
        q.set_backend(Backend.ONNXRUNTIME)
        q.enable_quant()
        q.enable_export_onnx()
    x = torch.randn(2, 8)
    # the export branch equals the stock fake-quantize ops (no native library involved: this runs on the CPU)
    torch.testing.assert_close(m.aq(x), torch.fake_quantize_per_tensor_affine(x, 0.05, 3, 0, 255))
    buf = io.BytesIO()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.onnx.export(m, (x,), buf, opset_version=13, dynamo=False)
    data = buf.getvalue()
    assert data.count(b"QuantizeLinear") >= 4 and data.count(b"DequantizeLinear") >= 2  # one Q / DQ pair per quantizer


@pytest.mark.skipif(not os.path.isdir("/root/reference/sparsebit"), reason="needs the reference checkout (build container only)")
def test_install_under_reference_quantmodel_resnet18_graph_build():
    """install() + the UNMODIFIED reference's QuantModel(torchvision resnet18): the fx graph build, operator
    replacement and quantizer construction still work with the native observers / runner / fake_quant module rebound
    (quant_model.py:185-189 imports the runner at call time)."""
    import subprocess
    import sys
    import textwrap

    code = textwrap.dedent("""
        import sys
        sys.path.insert(0, "tests/golden")
        import _ref_import as R
        R.install_shims()
        import torch, torchvision
        import sparsebit_b200
        sparsebit_b200.install()
        from sparsebit.quantization import QuantModel
        from sparsebit.quantization.quant_config import _C
        cfg = _C.clone(); cfg.DEVICE = "cpu"
        cfg.W.QSCHEME = "per-channel-symmetric"; cfg.W.QUANTIZER.BIT = 8
        cfg.A.QSCHEME = "per-tensor-affine"; cfg.A.QUANTIZER.BIT = 8
        qm = QuantModel(torchvision.models.resnet18(weights=None).eval(), cfg)
        qm.prepare_calibration()
        oprs = [m for m in qm.model.modules() if hasattr(m, "input_quantizer")]
        assert len(oprs) >= 40, len(oprs)
        assert type(qm.calibration_runner).__module__ == "sparsebit_b200.quantization.tools.calibration"
        native = [m for m in oprs if type(m.input_quantizer.observer).__module__.startswith("sparsebit_b200.")]
        assert len(native) == len(oprs)
        # LSQ of the reference keeps working on native observers: its constructor hook makes them retain batches
        cfg2 = _C.clone(); cfg2.DEVICE = "cpu"; cfg2.W.QSCHEME = "per-channel-symmetric"; cfg2.W.QUANTIZER.BIT = 4
        cfg2.W.QUANTIZER.TYPE = "lsq"; cfg2.A.QSCHEME = "per-tensor-affine"; cfg2.A.QUANTIZER.BIT = 4; cfg2.A.QUANTIZER.TYPE = "lsq"
        qm2 = QuantModel(torchvision.models.resnet18(weights=None).eval(), cfg2)
        lsq = [m.weight_quantizer for m in qm2.model.modules() if getattr(m, "weight_quantizer", None) is not None]
        assert lsq and all(q.observer.keep_data for q in lsq)
        print("GRAPH_OK", len(oprs))
    """)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip().splitlines()[-1].startswith("GRAPH_OK")
