"""CPU: the float64 references and value enumerations the element-by-element conv / Detect-head GPU tests rest on."""
import math

import numpy as np
import torch

from .conv_exact_ref import all_values, decode64, decode_bound, silu64, ulp


def test_ulp_matches_nextafter():
    """ulp(x) is the gap between |x| rounded down to the dtype and the next value up, for normals, subnormals and 0."""
    for dtype, tiny, sub in ((torch.float16, 2.0 ** -14, 2.0 ** -24), (torch.bfloat16, 2.0 ** -126, 2.0 ** -133)):
        v = all_values(dtype)
        f = v.double()
        f = f[(f > 0) & (f < f.max())]
        nxt = (v.view(torch.int16)[v.double() > 0].int() + 1)
        up = nxt.to(torch.int16).view(dtype).double()
        pos = v[v.double() > 0].double()
        keep = torch.isfinite(up) & (pos < pos.max())
        assert torch.equal(ulp(pos[keep], dtype), (up - pos)[keep])
        assert float(ulp(torch.tensor([0.0]), dtype)) == sub
        assert float(ulp(torch.tensor([tiny * 0.75]), dtype)) == sub
        assert float(ulp(torch.tensor([-tiny]), dtype)) == sub
        assert float(ulp(torch.tensor([1.0]), dtype)) == (2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7)
        assert float(ulp(torch.tensor([1.999]), dtype)) == (2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7)


def test_value_enumeration():
    h = all_values(torch.float16)
    assert h.numel() == 65536 - 2048  # every bit pattern but the 2 x 1024 with the all-ones exponent (inf / NaN)
    assert torch.isfinite(h.float()).all() and float(h.float().max()) == 65504.0
    assert len(set(h.view(torch.int16).tolist())) == h.numel()
    b = all_values(torch.bfloat16)
    assert b.numel() == 2 * 254 * 128 + 2  # exponents 1..254, both signs, 128 mantissas each, and +-0
    nz = b.float()[b.float() != 0].abs()
    assert float(nz.min()) == 2.0 ** -126 and torch.isfinite(b.float()).all()


def test_silu64_against_math():
    xs = [-1000.0, -745.0, -100.0, -20.0, -8.0, -1.0, -1e-30, 0.0, 1e-30, 0.5, 3.0, 30.0, 65504.0, 3.0e38]
    got = silu64(torch.tensor(xs, dtype=torch.float64)).tolist()
    for x, g in zip(xs, got):
        want = x / (1.0 + math.exp(-x)) if x > -700 else 0.0
        assert g == want or abs(g - want) <= 1e-15 * abs(want), (x, g, want)
    # the cancelling region the old epilogue form got wrong: silu(-8) = -8 / (1 + e^8)
    assert abs(float(silu64(torch.tensor([-8.0]))) + 2.682801e-3) < 1e-9


def test_decode64_against_a_direct_loop():
    g = torch.Generator().manual_seed(0)
    B, na, ny, nx, nc, nm = 2, 3, 4, 5, 2, 3
    no = 5 + nc + nm
    raw = torch.randn(B, na, ny, nx, no, generator=g, dtype=torch.float64) * 4
    anchors = torch.tensor([[10.0, 13.0], [16.0, 30.0], [33.0, 23.0]]) * 8
    z, grid = decode64(raw, nc, 8.0, anchors)
    r = raw.numpy()
    for b, a, y, x, o in np.ndindex(*raw.shape):
        v = r[b, a, y, x, o]
        s = 1.0 / (1.0 + math.exp(-v))
        want = {0: (2 * s + x - 0.5) * 8, 1: (2 * s + y - 0.5) * 8, 2: (2 * s) ** 2 * float(anchors[a, 0]),
                3: (2 * s) ** 2 * float(anchors[a, 1])}.get(o, s if o < 5 + nc else v)
        assert abs(float(z[b, a, y, x, o]) - want) <= 1e-12 * max(1.0, abs(want)), (b, a, y, x, o)
        assert float(grid[b, a, y, x, o]) == {0: x, 1: y}.get(o, 0)
    bound = decode_bound(z, grid, 8.0, torch.float16)
    assert (bound >= ulp(z, torch.float16)).all()
