"""rcp.approx.ftz.f32 and sqrt.approx.ftz.f32 -- the two hardware approximations on the TV-L1 engine's path (one MUFU
instruction each on sm_90a) -- as tables of their device values, and the rule that extends the tables to every float.
TEST INFRASTRUCTURE (see oracle/__init__.py).

The tables hold the device's values on [1, 2) (rcp, 2^23 entries) and [1, 4) (sqrt, 2^24 entries: mantissa x exponent
parity).  Everything else follows by scaling the exponent, with the .ftz rules:
  rcp:  +-0 and denormal inputs -> +-inf; +-inf -> +-0; NaN -> NaN; a result below FLT_MIN flushes to +-0;
  sqrt: +-0 and denormal inputs -> +-0; other negative inputs -> NaN; +inf -> +inf; NaN -> NaN.
oracle/tvl1_gpu_model.c (the "eng" build) applies the same rule in C; predict() states it in torch integer operations so
that it can be checked against the device on all 2^32 inputs (tests/test_tvl1_gpu.py).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

ONE_BITS = 0x3F800000
RCP_ENTRIES, SQRT_ENTRIES = 1 << 23, 1 << 24
OP_RCP, OP_SQRT = 0, 1


def table_inputs(op: int) -> np.ndarray:
    """The float32 inputs the table of `op` is taken at: [1, 2) for rcp, [1, 4) for sqrt, in bit order."""
    n = RCP_ENTRIES if op == OP_RCP else SQRT_ENTRIES
    return (np.arange(n, dtype=np.uint32) + np.uint32(ONE_BITS)).view(np.float32)


def correctly_rounded_tables():
    """Tables of the IEEE operations, 1/x and sqrt(x) rounded to nearest (the double result rounded to float is the
    correctly rounded float result for both)."""
    r = (1.0 / table_inputs(OP_RCP).astype(np.float64)).astype(np.float32)
    s = np.sqrt(table_inputs(OP_SQRT).astype(np.float64)).astype(np.float32)
    return r, s


def sample_inputs() -> np.ndarray:
    """Every exponent, both signs, 4096 mantissas each (both ends of the range, a stride and random ones): 2^21 float32
    inputs that reach every branch of the rule, the special values included."""
    rng = np.random.default_rng(11)
    mant = np.unique(np.concatenate([np.arange(0, 1 << 23, 1 << 12), np.arange(8), (1 << 23) - 1 - np.arange(8),
                                     rng.integers(0, 1 << 23, 2040)])).astype(np.uint32)
    bits = ((np.arange(256, dtype=np.uint32)[:, None] << 23) | mant[None, :]).ravel()
    return np.concatenate([bits, bits | np.uint32(0x80000000)]).view(np.float32)


def probe(op: int, x):
    """op applied on the device by the library's own rcp_approx / sqrt_approx (b2f_approx_probe) to a CUDA float32
    tensor; returns a new tensor."""
    import torch
    from opencv_contrib_b200 import _lib
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty_like(x)
    st = torch.cuda.current_stream(x.device)
    rc = _lib.lib().b2f_approx_probe(int(op), C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), x.numel(),
                                     C.c_void_p(st.cuda_stream))
    assert rc == 0, f"b2f_approx_probe returned {rc}"
    return out


@functools.lru_cache(maxsize=None)
def _device_tables(device: str):
    import torch
    out = []
    for op in (OP_RCP, OP_SQRT):
        x = torch.from_numpy(table_inputs(op)).to(device)
        out.append(probe(op, x).cpu().numpy())
    torch.cuda.synchronize(device)
    return tuple(out)


def device_tables(device):
    """(rcp table, sqrt table) as measured on `device`, float32 numpy arrays (cached per device)."""
    return _device_tables(str(device))


def predict(op: int, bits, rcp_tab, sqrt_tab):
    """The emulation in torch: int32 bit patterns in, int32 bit patterns of op(x) out.  rcp_tab / sqrt_tab: int32
    tensors of the tables' bits on the same device."""
    import torch
    sign = bits & -(1 << 31)
    e = (bits >> 23) & 0xFF
    m = bits & 0x7FFFFF
    nan = torch.full_like(bits, 0x7FC00000)
    if op == OP_RCP:
        y = rcp_tab[m.long()]
        ef = ((y >> 23) & 0xFF) - (e - 127)
        r = torch.where(ef > 0, sign | (ef.clamp(min=0) << 23) | (y & 0x7FFFFF), sign)
        r = torch.where(e == 0, sign | 0x7F800000, r)
        return torch.where(e == 0xFF, torch.where(m != 0, nan, sign), r)
    E = e - 127
    par = E & 1
    y = sqrt_tab[((par << 23) | m).long()]
    r = ((((y >> 23) & 0xFF) + ((E - par) >> 1)) << 23) | (y & 0x7FFFFF)
    r = torch.where(e == 0xFF, bits, r)
    r = torch.where(sign != 0, nan, r)
    return torch.where(e == 0, sign, r)
