"""Shared helpers for the parity tests."""
import math

import torch

from oracle import genie_oracle as O


class Guarded:
    """An output tensor placed `offset` elements into a buffer and followed by a guard of `guard` elements, all filled
    with a NaN bit pattern: an element the kernel never writes fails the comparison, and a write past the end changes
    the guard. `init` pre-fills the tensor itself (accumulated outputs start from non-zero values)."""
    BITS = {torch.bfloat16: (torch.int16, 0x7FA5), torch.float32: (torch.int32, 0x7FC0A5A5),
            torch.float64: (torch.int64, 0x7FF8A5A5A5A5A5A5)}

    def __init__(self, shape, dtype, guard=64, init=None, offset=0, device='cuda'):
        self.n = math.prod(shape) + offset
        self.buf = torch.empty(self.n + guard, dtype=dtype, device=device)
        ity, bits = self.BITS[dtype]
        self.buf.view(ity).fill_(bits)
        self.t = self.buf[offset:self.n].view(shape)
        if init is not None:
            self.t.copy_(init)

    def ptr(self):
        return self.t.data_ptr()

    def untouched(self):
        ity, bits = self.BITS[self.buf.dtype]
        return bool((self.buf.view(ity) == bits).all())

    def check_guard(self, name):
        ity, bits = self.BITS[self.buf.dtype]
        changed = int((self.buf[self.n:].view(ity) != bits).sum())
        assert changed == 0, f'{name}: {changed} guard elements after the tensor were overwritten'


def det_weights(module, gain=1.0):
    """Closed-form weights (the same ones oracle/make_golden.py loaded into the reference)."""
    shapes = {k: tuple(v.shape) for k, v in module.state_dict().items()}
    sd = O.det_state_dict(shapes, gain)
    missing = module.load_state_dict(sd, strict=False)
    assert all(k.endswith(('freq', 'bit_mask', 'blur')) for k in missing.missing_keys), missing
    return {k: v.detach().clone().cpu() for k, v in module.state_dict().items()}


def bf16_round(t):
    return t.to(torch.bfloat16).to(torch.float32)


def round_conv_weights(sd):
    """What the kernels see: conv / 5-D weights rounded to bf16, everything else fp32."""
    return {k: (bf16_round(v) if v.dim() == 5 else v) for k, v in sd.items()}


def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def assert_close(got, ref, rtol, atol, name=''):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    assert got.shape == ref.shape, f'{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    err = (got - ref).abs()
    bad = err > atol + rtol * ref.abs()
    if bad.any():
        i = torch.nonzero(bad.flatten())[0].item()
        raise AssertionError(f'{name}: {int(bad.sum())}/{bad.numel()} mismatches (rtol={rtol}, atol={atol}); '
                             f'max err {err.max().item():.3e}; first at flat {i}: got {got.flatten()[i].item():.6f} '
                             f'ref {ref.flatten()[i].item():.6f}')
