"""numpy restatement of the activation planes the tensor-core layers write (hand3d_b200/csrc/split_fmt.cuh, epilogue_store32 in
conv_wgmma.cu, the first-layer kernels in conv_direct.cu), bit for bit, and their decoders.

  bf16x3 / fp16x3   hi = rn16(v), lo = rn16(v - hi)            (v - hi in fp32, round to nearest even)
  bf16 / fp16       hi = rn16(v)
  fp16_f8c          h16 = fp16(clamp(32 v, +-65504)), l8 = e4m3_satfinite((v - h16 / 32) 2^10), h8 = e4m3_satfinite(v / 4)

bf16 and e4m3 conversions go through torch's CPU casts (round to nearest even); torch's float8_e4m3fn cast does not saturate (it
gives NaN past 448), so satfinite clamps to +-448 first, which rounds the same way because 448 is the largest finite e4m3.  The clamp
of the fp16 main plane uses fmin / fmax, as fminf / fmaxf do on the device (NaN-ignoring)."""
import numpy as np
import torch

f32, f64 = np.float32, np.float64
F16_MAX = 65504.0
E4M3_MAX = 448.0
F8C_MAIN, F8C_LO, F8C_HI = 32.0, 1024.0, 0.25   # kF8XMainScale, kF8XLoScale, kF8XHiScale
PLANES = {"bf16x3": ("hi", "lo"), "fp16x3": ("hi", "lo"), "bf16": ("hi",), "fp16": ("hi",), "fp16_f8c": ("hi", "l8", "h8")}
HALF = {"bf16x3": "bf16", "bf16": "bf16", "fp16x3": "fp16", "fp16": "fp16", "fp16_f8c": "fp16"}


def _f32(v):
    return np.ascontiguousarray(v, f32)


def bf16_bits(v):
    return torch.from_numpy(_f32(v)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def bf16_value(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(f32)


def fp16_bits(v):
    return _f32(v).astype(np.float16).view(np.uint16)


def fp16_value(bits):
    return np.asarray(bits, np.uint16).view(np.float16).astype(f32)


ENC16 = {"bf16": bf16_bits, "fp16": fp16_bits}
DEC16 = {"bf16": bf16_value, "fp16": fp16_value}


def split16(v, half):
    """(hi, lo) uint16 bits of the two-plane split."""
    v = _f32(v)
    hi = ENC16[half](v)
    lo = ENC16[half](v - DEC16[half](hi))
    return hi, lo


def split_ok(hi, lo, half):
    """The split invariant, element-wise: |lo| is at most half the spacing of the 16-bit format next to hi on lo's side, so
    rn16(hi + lo) == hi except where |lo| is exactly that half spacing (v - hi rounded to the midpoint; hi + lo then ties to even, which
    need not be hi).  A zero hi has a zero lo."""
    dec, enc = DEC16[half], ENC16[half]
    hi, lo = np.asarray(hi, np.uint16), np.asarray(lo, np.uint16)
    mag = hi & np.uint16(0x7FFF)
    h, l_ = dec(hi).astype(f64), dec(lo).astype(f64)
    up = dec(mag + np.uint16(1)).astype(f64) - dec(mag)
    down = dec(mag).astype(f64) - dec(np.maximum(mag, np.uint16(1)) - np.uint16(1))
    gap = np.where(np.sign(l_) == np.sign(h), up, down)
    ok = (np.abs(l_) <= gap / 2) & ((enc((h + l_).astype(f32)) == hi) | (np.abs(l_) == gap / 2))
    return np.where(h == 0, l_ == 0, ok)


def fp16_w_shift(colmax):
    """s(co) of the fp16 weight planes: max_k |w| 2^s in [2^13, 2^14), 0 for an all-zero (or NaN) column, clamped to [-126, 126]."""
    colmax = np.asarray(colmax, f32)
    _, e = np.frexp(colmax)
    s = np.clip(14 - e.astype(np.int64), -126, 126)
    return np.where(colmax > 0, s, 0)


def e4m3_bits(v):
    """e4m3 with __NV_SATFINITE: round to nearest even, finite values past 448 saturate."""
    return torch.from_numpy(np.clip(_f32(v), -E4M3_MAX, E4M3_MAX)).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def e4m3_value(bits):
    return torch.from_numpy(np.ascontiguousarray(bits, np.uint8)).view(torch.float8_e4m3fn).to(torch.float32).numpy()


def f8c_planes(v):
    """(h16, l8, h8) of f32_to_f8c."""
    v = _f32(v)
    h16 = fp16_bits(np.fmin(np.fmax(v * f32(F8C_MAIN), f32(-F16_MAX)), f32(F16_MAX)))
    l8 = e4m3_bits((v - fp16_value(h16) * f32(1.0 / F8C_MAIN)) * f32(F8C_LO))
    h8 = e4m3_bits(v * f32(F8C_HI))
    return h16, l8, h8


def f8c_value(h16, l8):
    """h16 / 32 + l8 / 1024 (exact in fp64)."""
    return fp16_value(h16).astype(f64) / F8C_MAIN + e4m3_value(l8).astype(f64) / F8C_LO


def encode(v, precision):
    """The planes a layer of `precision` stores for the fp32 values v: {"hi": uint16, "lo": uint16, "l8": uint8, "h8": uint8},
    holding only the planes of the format."""
    if precision == "fp16_f8c":
        h16, l8, h8 = f8c_planes(v)
        return {"hi": h16, "l8": l8, "h8": h8}
    half = HALF[precision]
    if precision in ("bf16", "fp16"):
        return {"hi": ENC16[half](v)}
    hi, lo = split16(v, half)
    return {"hi": hi, "lo": lo}


def decode(planes, precision):
    """fp64 value the next layer's operands represent (hi + lo, hi, or h16 / 32 + l8 / 1024)."""
    if precision == "fp16_f8c":
        return f8c_value(planes["hi"], planes["l8"])
    dec = DEC16[HALF[precision]]
    v = dec(planes["hi"]).astype(f64)
    if "lo" in PLANES[precision]:
        v = v + dec(planes["lo"])
    return v


# relative resolution of each format's decoded value (half an ulp of the last plane, with margin) and the absolute floor below which
# its last plane is subnormal; decoded planes are held to |decode - ref| <= BOUND S + REL |ref| + ABS
FORMAT_REL = {"bf16x3": 2.0 ** -16, "fp16x3": 2.0 ** -21, "bf16": 2.0 ** -8, "fp16": 2.0 ** -11, "fp16_f8c": 2.0 ** -14}
FORMAT_ABS = {"bf16x3": 0.0, "fp16x3": 2.0 ** -25, "bf16": 0.0, "fp16": 2.0 ** -25, "fp16_f8c": 2.0 ** -20}
