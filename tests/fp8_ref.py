# coding=utf-8
"""numpy restatement of the fp8 message-row format of include/tfgk.h (e4m3fn bytes, one power-of-two exponent per row and
group of 128 columns).  The exponent is derived in float64 and the bytes come from torch's round-to-nearest-even cast of
the float64 scaled values, independently of the kernels' bit tricks."""
import numpy as np
import torch

E4M3_MAX = 448.0


def exponent(m):
    """Smallest integer k with m * 2^-k <= 448, clamped to [-126, 127]; 0 for m == 0 (m = max |x| over finite x)."""
    m = float(m)
    if m == 0.0:
        return 0
    k = int(np.ceil(np.log2(m / E4M3_MAX)))
    while m * 2.0 ** -k > E4M3_MAX:
        k += 1
    while m * 2.0 ** -(k - 1) <= E4M3_MAX:
        k -= 1
    return max(-126, min(127, k))


def quantize(x, group=128):
    """x [R, C] float32 -> (bytes uint8 [R, C], exps int8 [R, ceil(C / 128)])."""
    x = np.asarray(x, dtype=np.float32)
    R, C = x.shape
    G = max(-(-C // group), 1)
    q = np.zeros((R, C), np.uint8)
    ks = np.zeros((R, G), np.int8)
    x64 = x.astype(np.float64)
    for g in range(G):
        blk = x64[:, g * group:(g + 1) * group]
        fin = np.where(np.isfinite(blk), np.abs(blk), 0.0)
        for r in range(R):
            k = exponent(fin[r].max() if fin.shape[1] else 0.0)
            ks[r, g] = k
            scaled = blk[r] * 2.0 ** -k
            q[r, g * group:(g + 1) * group] = torch.from_numpy(scaled).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    return q, ks


def dequantize(q, ks, group=128):
    """x^ = float(q) * 2^k as float32: exact, except that a value that rounded up past FLT_MAX becomes inf."""
    q = np.asarray(q, np.uint8)
    R, C = q.shape
    v = torch.from_numpy(np.ascontiguousarray(q)).view(torch.float8_e4m3fn).to(torch.float64).numpy()
    k = np.repeat(np.asarray(ks, np.float64), group, axis=1)[:, :C] if C else np.zeros((R, 0))
    with np.errstate(over="ignore"):
        return (v * 2.0 ** k).astype(np.float32)


def error_bound(x, ks, group=128):
    """Per-element bound max(2^-4 |x|, 2^(k-10)) of |x^ - x| for finite x."""
    x = np.asarray(x, np.float64)
    k = np.repeat(np.asarray(ks, np.float64), group, axis=1)[:, :x.shape[1]]
    return np.maximum(np.abs(x) * 2.0 ** -4, 2.0 ** (k - 10))
