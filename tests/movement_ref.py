"""Device-free references for the data-movement kernels (SPPF pooling forward and backward, 2x nearest upsample and its
backward, zero stuffing, stem space-to-depth, NHWC -> NCHW export), written as plain torch / numpy expressions.  Every
function works on the device of its input; float64 max_pool2d runs torch's NCHW kernel, whose arg-max rule (first
maximum in row-major window order, a NaN replaces the running maximum so the last NaN wins) is the rule the engine's
backward implements."""
import numpy as np
import torch
import torch.nn.functional as F


def bit_patterns(shape, dtype: torch.dtype, seed: int = 0) -> torch.Tensor:
    """Every 16-bit pattern (NaN payloads, +-inf, subnormals, -0 included) in a seeded permutation, tiled to `shape`, as
    `dtype` (fp16 or bf16) on the CPU.  Shapes of at least 65536 elements contain each pattern at least once."""
    g = torch.Generator().manual_seed(seed)
    n = int(np.prod(shape))
    perm = (torch.randperm(65536, generator=g) - 32768).to(torch.int16)
    return perm.repeat((n + 65535) // 65536)[:n].view(dtype).reshape(shape)


def sppf_fwd(x: torch.Tensor, k: int):
    """SPPF's pooling chain y1 = m(x), y2 = m(y1), y3 = m(y2), m = max_pool2d(k, 1, k // 2), in float64 (NCHW)."""
    x = x.double().contiguous()
    y1 = F.max_pool2d(x, k, 1, k // 2)
    y2 = F.max_pool2d(y1, k, 1, k // 2)
    y3 = F.max_pool2d(y2, k, 1, k // 2)
    return y1, y2, y3


def sppf_bwd(a: torch.Tensor, dcat: torch.Tensor, k: int) -> torch.Tensor:
    """d/da of cat(a, y1, y2, y3) . dcat (dcat (B, 4c, H, W)) by float64 autograd through sppf_fwd."""
    x = a.detach().to(torch.float64, copy=True).contiguous().requires_grad_(True)
    cat = torch.cat((x, *sppf_fwd(x, k)), 1)
    cat.backward(dcat.double().contiguous())
    return x.grad


def windowed_max(x: torch.Tensor, win: int) -> torch.Tensor:
    """max over the clipped win x win window centred on each pixel (stride 1, pad win // 2), float64, NaN-propagating."""
    return F.max_pool2d(x.double().contiguous(), win, 1, win // 2)


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    """nearest 2x upsample (B, C, H, W) -> (B, C, 2H, 2W) as an index expression (bit copy, any dtype)."""
    return x.repeat_interleave(2, 2).repeat_interleave(2, 3)


def upsample2x_bwd_f32(dy: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """The upsample backward in the kernel's documented order, emulated in numpy float32: acc = 0, then acc += dy at
    (0,0), (0,1), (1,0), (1,1) of each 2x2 block, then one round-to-nearest-even into `dtype`."""
    d = dy.float().cpu().numpy()
    acc = np.zeros(d[:, :, 0::2, 0::2].shape, np.float32)
    for oy, ox in ((0, 0), (0, 1), (1, 0), (1, 1)):
        acc = acc + d[:, :, oy::2, ox::2]
    return torch.from_numpy(acc).to(dtype)


def upsample2x_bwd64(dy: torch.Tensor) -> torch.Tensor:
    """The upsample backward as a float64 sum of each 2x2 block."""
    d = dy.double()
    return d[:, :, 0::2, 0::2] + d[:, :, 0::2, 1::2] + d[:, :, 1::2, 0::2] + d[:, :, 1::2, 1::2]


def zero_stuff2x(x: torch.Tensor) -> torch.Tensor:
    """(B, C, H, W) -> (B, C, 2H, 2W) with x at the even (y, x) positions and +0 elsewhere (any dtype)."""
    b, c, h, w = x.shape
    z = torch.zeros(b, c, 2 * h, 2 * w, dtype=x.dtype, device=x.device)
    z[:, :, 0::2, 0::2] = x
    return z


def stem_s2d(img: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """(B, 3, H, W) image -> (B, H/2, W/2, 16) NHWC: input pixel (2i + dy, 2j + dx) of colour c lands in channel
    (dy*2 + dx)*3 + c of cell (i, j); channels 12..15 are +0.  uint8 is float32 x / 255 rounded to nearest even, every
    other input dtype is `.float().to(dtype)`."""
    if img.dtype == torch.uint8:  # numpy's float32 division is correctly rounded (torch may multiply by a reciprocal)
        v = torch.from_numpy(img.cpu().numpy().astype(np.float32) / np.float32(255)).to(img.device)
    else:
        v = img.float()
    v = v.to(dtype)
    b, _, h, w = img.shape
    out = torch.zeros(b, h // 2, w // 2, 16, dtype=dtype, device=img.device)
    for dy in range(2):
        for dx in range(2):
            for c in range(3):
                out[..., (dy * 2 + dx) * 3 + c] = v[:, c, dy::2, dx::2]
    return out


def nhwc_to_nchw(x: torch.Tensor) -> torch.Tensor:
    """(B, H, W, C) -> dense (B, C, H, W), element (n, c, y, x) = x[n, y, x, c]."""
    return x.permute(0, 3, 1, 2).contiguous()
