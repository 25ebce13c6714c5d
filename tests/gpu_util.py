import zlib

import numpy as np
import pytest
import torch

from sparsebit_b200 import _lib


def _tf32_off():
    """TF32 off for cuDNN convs and cuBLAS matmuls over a test, so that the fp32 comparison paths round as fp32."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ``no_tf32`` for the tests that ask for it; a module that imports ``no_tf32_autouse`` has it on every test
no_tf32 = pytest.fixture(_tf32_off, name="no_tf32")
no_tf32_autouse = pytest.fixture(_tf32_off, autouse=True, name="no_tf32_autouse")


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def bits_equal(a, b):
    """Bit-exact float comparison up to the sign of zero (SURVEY Q17) with NaN == NaN."""
    a = np.asarray(a, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    if a.shape != b.shape:
        return False
    return np.array_equal(np.where(a == 0, 0.0, a), np.where(b == 0, 0.0, b), equal_nan=True)


def t(x, device=None):
    return torch.from_numpy(np.ascontiguousarray(x)).to(device or dev())


def on_device(a, offset=0, *, unit="elem"):
    """A device copy of ``a`` that starts ``offset`` elements (``unit="byte"``: bytes) into a fresh zeroed allocation,
    which the caching allocator aligns to at least 16 bytes, with at least 16 bytes of slack behind it."""
    assert unit in ("elem", "byte"), unit
    a = np.array(a, order="C")
    byte_off = offset * a.itemsize if unit == "elem" else offset
    raw = torch.zeros(byte_off + a.nbytes + 16, dtype=torch.uint8, device=dev())
    view = raw[byte_off:byte_off + a.nbytes].view(torch.from_numpy(a.reshape(-1)[:0]).dtype).view(a.shape)
    view.copy_(torch.from_numpy(a))
    return view


def stream():
    return torch.cuda.current_stream().cuda_stream


def real_sm():
    return int(_lib.load().sb200_sm_count())


def seed(name):
    return zlib.crc32(name.encode())


def seed_of(name, *extra):
    return zlib.crc32(repr((name,) + extra).encode())
