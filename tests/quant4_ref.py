"""Restatement of bitsandbytes 4-bit weights (FP4 / NF4, blocksize 64) in torch, fp32 on the CPU.

Follows bitsandbytes 0.39-0.41 quantize_4bit / dequantize_4bit / MatMul4Bit as include/seedb200.h states them.
bitsandbytes is not a dependency of this project, so this restatement is not checked against bitsandbytes itself.
"""
import torch

FP4, NF4 = 0, 1
BLOCK = 64

NF4_VALUES = torch.tensor([-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
                           -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
                           0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941,
                           0.7229568362236023, 1.0], dtype=torch.float32)
# fp32 midpoints of adjacent NF4 values: a normalised value strictly above k of them gets code k
NF4_THRESHOLDS = (NF4_VALUES[:-1] + NF4_VALUES[1:]) * 0.5

_FP4_MAG = torch.tensor([0.0, 0.005208333333, 0.66666667, 1.0, 0.33333333, 0.5, 0.16666667, 0.25], dtype=torch.float32)
FP4_VALUES = torch.cat([_FP4_MAG, -_FP4_MAG])               # bit 8 = sign (code 8 is -0.0)
FP4_PIVOTS = torch.tensor([0.00260417, 0.0859375, 0.20833333, 0.29166667, 0.4166667, 0.583333, 0.8333333],
                          dtype=torch.float32)
FP4_BUCKET_CODE = torch.tensor([0b000, 0b001, 0b110, 0b111, 0b100, 0b101, 0b010, 0b011])


def values(qt):
    return FP4_VALUES if qt == FP4 else NF4_VALUES


def absmax(w):
    """fp16 [N, K] -> fp32 [N, K/64]: max |w| per block, NaN dropped (fmaxf)"""
    a = w.float().abs().reshape(w.shape[0], -1, BLOCK)
    return torch.where(torch.isnan(a), torch.zeros_like(a), a).amax(-1)


def codes(n, qt):
    """normalised fp32 values -> 4-bit codes (int64)"""
    if qt == NF4:
        return (n[..., None] > NF4_THRESHOLDS).sum(-1)
    bucket = (n.abs()[..., None] > FP4_PIVOTS).sum(-1)
    return FP4_BUCKET_CODE[bucket] | torch.where(n < 0, 8, 0)


def pack(c):
    """codes [N, K] -> uint8 [N, K/2], the even-index element in the high nibble"""
    return ((c[:, 0::2] << 4) | c[:, 1::2]).to(torch.uint8)


def unpack(packed):
    p = packed.long()
    return torch.stack([p >> 4, p & 15], -1).reshape(packed.shape[0], -1)


def quantize(w, qt, rows=1024):
    """fp16 [N, K] (K % 64 == 0) -> (packed uint8 [N, K/2], absmax fp32 [N, K/64]); `rows` bounds the work per step"""
    N, K = w.shape
    assert K % BLOCK == 0
    am = absmax(w)
    packed = torch.empty((N, K // 2), dtype=torch.uint8)
    for r0 in range(0, N, rows):
        blk = w[r0:r0 + rows].float().reshape(-1, K // BLOCK, BLOCK)
        n = blk * (1.0 / am[r0:r0 + rows])[..., None]         # correctly rounded fp32 reciprocal, then one product
        packed[r0:r0 + rows] = pack(codes(n, qt).reshape(-1, K))
    return packed, am


def dequantize(packed, am, qt):
    """-> W' fp16 [N, K] = fp16_rn(value[code] * absmax)"""
    N = packed.shape[0]
    v = values(qt)[unpack(packed)].reshape(N, -1, BLOCK)
    return (v * am[..., None]).reshape(N, -1).half()


def linear4(x, packed, am, qt, residual=None):
    """MatMul4Bit: fp16(x . W'^T) with fp32 accumulation (+ residual, rounded again)"""
    y = (x.float() @ dequantize(packed, am, qt).float().t()).half()
    if residual is not None:
        y = (y.float() + residual.float()).half()
    return y
