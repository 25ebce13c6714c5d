"""Integer-grid convs with a DoReFa input (the DoReFa QAT recipe, 4-bit weights and activations) against the fake-quant
DoReFa conv, on every conv of ResNet-18, ResNet-50 and MobileNetV2 (torchvision, 224 x 224 input) at batch 256, plus
ResNet-50 under the PACT recipe (DoReFa weights, a plain 4-bit unsigned activation grid).

Per stack, one JSON line (times in ms, summed over the stack's convs, the median and [min, max] of three alternated
repeats, CUDA events over repeated calls after warm-up), and per conv one line with the same arms in us:
  fq_f32, fq_tf32   -- the fake-quant layer: DoReFaSTE on x (or the plain QDQ for PACT), the fake-quant weight, then
                       cuDNN F.conv2d, TF32 off / on;
  int8_nchw         -- the converted layer on an NCHW input (for DoReFa: dorefa_absmax, then the _dorefa entry point);
  int8_nhwc         -- the converted layer on a channels-last input;
  plain_nchw, plain_nhwc -- the same layer with a uniform input quantizer: what the abs-max pass and tanhf in the
                       lowering cost.
Each converted conv, DoReFa and uniform input, is checked against its fake-quant layer in the run: NaN positions equal,
within 2^-21 (conv(|fx|, |fw|) + |bias|) of the fp64 conv of the fake-quant operands, and its channels-last output
equal to the NCHW one bit for bit.  The card name and power limit are read
in the same run.  Usage: python scripts/bench_int8_dorefa.py [--quick]"""
import collections
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch
import torch.nn as nn
import torch.nn.functional as F

from bench_int8_conv_nhwc import model_convs
from bench_util import card, set_tf32, timeit
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.modules import QConv2d, from_dorefa_adaround

CL = torch.channels_last


def _layer(geom, x, a_type):
    """A calibrated QConv2d of geometry ``geom``: 4-bit ``a_type`` input (per-tensor), 4-bit DoReFa weight
    (per-channel symmetric), MinMax qparams from ``x``."""
    c_in, _, _, c_out, groups, k, stride, padding, dilation = geom
    conv = nn.Conv2d(c_in, c_out, k, stride=stride, padding=padding, dilation=dilation, groups=groups).cuda()
    q = QConv2d(conv).build_quantizer(sbcfg.quantizer_config("per-tensor-affine", 4, "feature", qtype=a_type),
                                      sbcfg.quantizer_config("per-channel-symmetric", 4, "weight", qtype="dorefa"))
    q = q.cuda().eval()
    for quantizer, v in ((q.input_quantizer, x), (q.weight_quantizer, q.weight)):
        quantizer.update_observer(v.detach())
        quantizer.calc_qparams()
    q.set_quant(w_quant=True, a_quant=True)
    return q


def _check(y, mod, x):
    with torch.no_grad():
        fx, fw = mod.input_quantizer(x).double(), mod.weight_quantizer(mod.weight).double()
        b = mod.bias.double()
        t = F.conv2d(fx, fw, b, **mod.fwd_kwargs)
        a = F.conv2d(fx.abs(), fw.abs(), b.abs(), **mod.fwd_kwargs)
    ok = ~torch.isnan(t)
    return bool(torch.equal(torch.isnan(y), torch.isnan(t))) and bool(
        ((y.double() - t).abs()[ok] <= 2.0 ** -21 * a[ok] + 1e-30).all())


def alternated(arms, repeats=3):
    times = collections.defaultdict(list)
    for _ in range(repeats):
        for name, (tf32, fn) in arms.items():
            set_tf32(tf32)
            times[name].append(timeit(fn, budget_s=0.1))
    set_tf32(False)
    return {k: (statistics.median(v), min(v), max(v)) for k, v in times.items()}


def bench_conv(geom, n, a_type):
    c_in, h, w = geom[:3]
    torch.manual_seed(sum(geom) + n)
    x = torch.randn(n, c_in, h, w, device="cuda")
    xc = x.to(memory_format=CL)
    fq, fq_plain = _layer(geom, x, a_type), _layer(geom, x, "uniform")
    conv, plain = from_dorefa_adaround(fq), from_dorefa_adaround(fq_plain)
    with torch.no_grad():
        ok = True
        for layer, ref in ((conv, fq), (plain, fq_plain)):
            y = layer(x)
            ok &= _check(y, ref, x) and torch.equal(layer(xc).contiguous().view(torch.int32), y.view(torch.int32))
        arms = {"fq_f32": (False, lambda: fq(x)), "fq_tf32": (True, lambda: fq(x)),
                "int8_nchw": (False, lambda: conv(x)), "int8_nhwc": (False, lambda: conv(xc)),
                "plain_nchw": (False, lambda: plain(x)), "plain_nhwc": (False, lambda: plain(xc))}
        stats = alternated(arms)
    del x, xc
    return stats, ok


def main():
    quick = "--quick" in sys.argv
    info = card()
    n = 32 if quick else 256
    stacks = [("resnet18", "dorefa"), ("resnet50", "dorefa"), ("mobilenet_v2", "dorefa"), ("resnet50", "pact")]
    for family, a_type in stacks[:1] if quick else stacks:
        convs = model_convs(family)
        totals = collections.defaultdict(lambda: [0.0, 0.0, 0.0])
        all_ok = True
        for i, geom in enumerate(convs):
            stats, ok = bench_conv(geom, n, a_type)
            all_ok &= ok
            rec = {"stack": family, "recipe": a_type, "conv": i, "geom": list(geom), "batch": n, "checked": ok, **info}
            for k, (med, lo, hi) in stats.items():
                rec[k + "_us"] = round(med, 2)
                rec[k + "_range_us"] = [round(lo, 2), round(hi, 2)]
                for j, v in enumerate((med, lo, hi)):
                    totals[k][j] += v / 1e3
            print(json.dumps(rec), flush=True)
            torch.cuda.empty_cache()
        rec = {"stack": family, "recipe": a_type, "convs": len(convs), "batch": n, "checked": all_ok, **info}
        for k, (med, lo, hi) in totals.items():
            rec[k + "_ms"] = round(med, 3)
            rec[k + "_range_ms"] = [round(lo, 3), round(hi, 3)]
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
