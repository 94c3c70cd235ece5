"""Device-free references for the element-by-element conv / Detect-head tests: the unit in the last place of a value in fp16 or
bf16, every finite fp16 and every normal bf16 value, and float64 SiLU and Detect decode."""
import torch

# (mantissa bits after the point, smallest normal exponent) of each output dtype
_FMT = {torch.float16: (10, -14), torch.bfloat16: (7, -126)}


def ulp(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """float64 spacing of `dtype` at |x| (x float64): 2^(e - mantissa bits) with e = floor(log2|x|), clamped to the smallest normal
    exponent, so below the smallest normal (and at 0) it is the subnormal step."""
    man, emin = _FMT[dtype]
    x = x.double().abs()
    _, e = torch.frexp(x)  # |x| = m * 2^e, m in [0.5, 1)  ->  floor(log2|x|) = e - 1
    e = torch.where(x > 0, e - 1, torch.full_like(e, emin)).clamp_min(emin)
    return torch.ldexp(torch.ones_like(x), (e - man).to(torch.int32))


def all_values(dtype: torch.dtype) -> torch.Tensor:
    """Every finite fp16 value (subnormals and both zeros included), or every normal bf16 value plus both zeros, as `dtype`."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    v = bits.view(dtype)
    f = v.float()
    keep = torch.isfinite(f)
    if dtype == torch.bfloat16:
        keep &= (f.abs() >= 2.0 ** -126) | (f == 0)
    return v[keep]


def silu64(x: torch.Tensor) -> torch.Tensor:
    """x * sigmoid(x) in float64 (x / (1 + e^-x); e^-x overflows to inf for x < -709 and the quotient to -0, as it should)."""
    x = x.double()
    return x / (1.0 + torch.exp(-x))


def sigmoid64(x: torch.Tensor) -> torch.Tensor:
    x = x.double()
    return 1.0 / (1.0 + torch.exp(-x))


def decode64(raw: torch.Tensor, nc: int, stride: float, anchor_wh: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Detect decode (models/yolo.py Detect) of raw logits (B, na, ny, nx, no) in float64: sigmoid for box / conf / class columns,
    xy = (2 sigma + grid - 0.5) * stride, wh = (2 sigma)^2 * anchor (pixels), columns >= 5 + nc passed through.
    Returns (z (B, na, ny, nx, no), |grid| per element: the grid coordinate of the xy columns, 0 elsewhere)."""
    raw = raw.double()
    _, na, ny, nx, no = raw.shape
    s = sigmoid64(raw)
    gy, gx = torch.meshgrid(torch.arange(ny, dtype=torch.float64, device=raw.device),
                            torch.arange(nx, dtype=torch.float64, device=raw.device), indexing="ij")
    z = raw.clone()
    z[..., 4 : 5 + nc] = s[..., 4 : 5 + nc]
    z[..., 0] = (2 * s[..., 0] + gx - 0.5) * stride
    z[..., 1] = (2 * s[..., 1] + gy - 0.5) * stride
    anc = anchor_wh.double().to(raw.device).view(1, na, 1, 1, 2)
    z[..., 2:4] = (2 * s[..., 2:4]) ** 2 * anc
    grid = torch.zeros_like(raw)
    grid[..., 0] = gx
    grid[..., 1] = gy
    return z, grid


def decode_bound(z64: torch.Tensor, grid: torch.Tensor, stride: float, dtype: torch.dtype) -> torch.Tensor:
    """Per-element bound on |z - z64|: the dtype's ulp at the result plus the fp32 arithmetic of the xy decode
    (2^-20 * (|grid| + 2) * stride)."""
    return ulp(z64, dtype) + 2.0 ** -20 * (grid.abs() + 2) * stride
