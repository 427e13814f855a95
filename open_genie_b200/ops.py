"""Autograd-aware Python bindings of the CUDA hot path (everything goes through the C ABI in _lib).

Internal tensor convention ("internal format"): a video is a torch tensor with the reference's LOGICAL
shape (B, C, T, H, W) whose memory is NDHWC (channels-last-3d) — bf16 between kernels, fp32 for the few
tensors that feed a loss (encoder head -> LFQ, decoder tail -> mse). `to_internal` / `to_reference`
convert at the public boundary (the reference is NCDHW fp32 everywhere, e.g. genie/tokenizer.py:307-330).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _lib

bf16 = torch.bfloat16
f32 = torch.float32


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------
# step-scoped zero arena + split-K workspace, both owned by a "step scope"
# ------------------------------------------------------------------------------------------------
def _in_backward() -> bool:
    """True while autograd is executing a backward graph on this thread (custom Function.backward runs with grad
    mode OFF, so torch.is_grad_enabled() cannot tell a backward pass from a no_grad forward)."""
    return torch._C._current_graph_task_id() != -1


class ZeroArena:
    """Bump allocator for the zero-initialised accumulators of ONE training step (the fp32 buffers the weight-
    gradient kernel reduces into, bias / gamma / beta gradients, GroupNorm sums and reduction buffers): one fill of
    the extent used by the previous step replaces ~540 small fill launches, and — because every parameter gradient
    of the step then lives in one contiguous range — the data-parallel all-reduce runs directly on slices of it
    (ddp.ArenaGradAllReducer): no bucket copies.

    Lifetime contract: everything handed out is valid until the first allocation after the next `mark_step()`
    (FusedAdamW.step() calls it), so gradients must be released with `zero_grad(set_to_none=True)` every step.
    Only allocations made while a gradient can exist are served (grad mode on, or inside backward); a no_grad /
    inference forward gets plain torch.zeros, so it can never see or disturb a step's accumulators.

    Memory is a list of segments: the first step of a model grows it segment by segment; the next step boundary
    consolidates it into one buffer (never while a CUDA graph is being captured, and never again once `frozen` —
    a captured graph has the addresses baked in)."""

    SEGMENT = 256 << 20

    def __init__(self):
        self.segs = {}       # device -> [uint8 tensors]
        self.cur = {}        # device -> (segment index, byte offset) of the next allocation
        self.hi = {}         # device -> [bytes used per segment] in the current step
        self.bwd0 = {}       # device -> (segment, offset) of the first allocation made inside backward this step
        self.dirty = {}      # device -> a step boundary passed since the last allocation
        self.frozen = False
        self.generation = 0  # step boundaries passed: a value kept with an arena tensor tells whether it may be stale

    # -- step boundary ---------------------------------------------------------------------------
    def mark_step(self):
        self.generation += 1
        for d in self.dirty:
            self.dirty[d] = True

    def _begin(self, dev):
        segs = self.segs.setdefault(dev, [])
        used = self.hi.get(dev, [])
        capturing = dev.type == 'cuda' and torch.cuda.is_current_stream_capturing()
        if len(segs) > 1 and not capturing and not self.frozen:
            total = sum(used)
            segs[:] = [torch.zeros(min(int(total * 1.05) + (1 << 20), 32 << 30), dtype=torch.uint8, device=dev)]
        else:
            for t, u in zip(segs, used):
                if u:
                    t[:u].zero_()
        self.cur[dev] = (0, 0)
        self.hi[dev] = [0] * len(segs)
        self.bwd0.pop(dev, None)
        self.dirty[dev] = False

    # -- allocation ------------------------------------------------------------------------------
    def zeros(self, shape, dtype, device):
        dev = torch.device(device)
        if dev.type == 'cuda' and dev.index is None:
            dev = torch.device('cuda', torch.cuda.current_device())
        if self.dirty.setdefault(dev, True):
            self._begin(dev)
        n = 1
        for d in (shape if isinstance(shape, (tuple, list, torch.Size)) else (shape,)):
            n *= int(d)
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        if nbytes == 0:
            return torch.zeros(shape, dtype=dtype, device=dev)
        al = (nbytes + 255) & ~255
        segs, hi = self.segs[dev], self.hi[dev]
        si, off = self.cur[dev]
        while si < len(segs) and off + al > segs[si].numel():
            si, off = si + 1, 0
        if si == len(segs):
            capturing = dev.type == 'cuda' and torch.cuda.is_current_stream_capturing()
            if self.frozen or capturing:
                raise RuntimeError('open_genie_b200: the zero arena of a captured training step is too small for this '
                                   'step (shapes changed after capture?) — re-create the GraphedTrainStep')
            segs.append(torch.zeros(max(self.SEGMENT, al), dtype=torch.uint8, device=dev))   # fresh: already zero
            hi.append(0)
        if dev not in self.bwd0 and _in_backward():
            self.bwd0[dev] = (si, off)
        self.cur[dev] = (si, off + al)
        hi[si] = off + al
        return segs[si][off:off + nbytes].view(dtype).view(shape)

    # -- introspection (ddp.ArenaGradAllReducer, tests) ------------------------------------------
    def position(self, dev):
        return self.cur.get(torch.device(dev), (0, 0))

    def locate(self, t: Tensor):
        """(segment, byte offset) of tensor `t` if its storage lies inside this arena, else None."""
        p = t.data_ptr()
        for si, s in enumerate(self.segs.get(t.device, [])):
            o = p - s.data_ptr()
            if 0 <= o < s.numel():
                return si, o
        return None

    def bytes_in_use(self, dev=None):
        return sum(sum(v) for d, v in self.hi.items() if dev is None or d == torch.device(dev))


class StepScope:
    """The mutable scratch a training step's kernels use: the zero arena and the split-K workspace. The process has
    one default scope (arena off unless enable_zero_arena()); a GraphedTrainStep owns a PRIVATE scope that is never
    reallocated or freed while its graph is alive, so eager calls made later (validation, tokenize(), a bigger
    batch) cannot free or overwrite memory whose address is baked into the captured graph."""

    def __init__(self, arena: Optional[ZeroArena] = None):
        self.arena = arena
        self.ws = {}          # device -> uint8 workspace
        self.scratch_bufs = {}   # device -> uint8 scratch for per-block / per-split partial sums (no contents kept)
        self.frozen = False

    SCRATCH_BYTES = 64 << 20

    def scratch(self, dev):
        """Scratch for the reproducible reductions (weight-gradient partial tiles, GroupNorm backward partials): every
        use is stream-ordered and complete inside one C-ABI call; the kernels limit their split to what fits."""
        t = self.scratch_bufs.get(dev)
        if t is None:
            if self.frozen or (dev.type == 'cuda' and torch.cuda.is_current_stream_capturing()):
                raise RuntimeError('open_genie_b200: reduction scratch of a captured training step would have to grow')
            t = torch.empty(self.SCRATCH_BYTES, dtype=torch.uint8, device=dev)
            self.scratch_bufs[dev] = t
        return t

    def workspace(self, dev, nbytes: int):
        # >= 24 MB: room for one partial-sum slab per split (splits x tiles <= 132 tiles of 128 x 128 fp32 = 8.7 MB)
        nbytes = min(max(nbytes, 24 << 20), 1 << 30)
        t = self.ws.get(dev)
        if t is None or t.numel() < nbytes:
            if self.frozen or (dev.type == 'cuda' and torch.cuda.is_current_stream_capturing()):
                raise RuntimeError('open_genie_b200: split-K workspace of a captured training step would have to grow')
            t = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            self.ws[dev] = t
        return t

    def freeze(self):
        self.frozen = True
        if self.arena is not None:
            self.arena.frozen = True


_DEFAULT_SCOPE = StepScope()
_SCOPE = _DEFAULT_SCOPE
ZERO_ARENA = ZeroArena()      # the default scope's arena when enable_zero_arena(True)


class step_scope:
    """`with ops.step_scope(scope): ...` — route arena / workspace allocations to `scope`."""

    def __init__(self, scope: StepScope):
        self.scope = scope

    def __enter__(self):
        global _SCOPE
        self.prev, _SCOPE = _SCOPE, self.scope
        return self.scope

    def __exit__(self, *exc):
        global _SCOPE
        _SCOPE = self.prev
        return False


def enable_zero_arena(on: bool = True):
    """Opt in to the step-scoped zero arena for eagerly launched training steps (see ZeroArena for the contract)."""
    _DEFAULT_SCOPE.arena = ZERO_ARENA if on else None


def current_arena() -> Optional[ZeroArena]:
    return _SCOPE.arena


def mark_step():
    """A training step ended (gradients consumed): the current scope's arena may be recycled."""
    if _SCOPE.arena is not None:
        _SCOPE.arena.mark_step()


def _zeros(shape, dtype, device, recording: bool = False):
    """Zero-initialised accumulator. Served from the step's arena only while a gradient can exist: inside backward, in
    grad mode, or — `recording` — inside the forward of an autograd Function that is being recorded (Function.forward
    itself runs with grad mode off; its ctx.needs_input_grad tells a training forward from a no_grad / inference one)."""
    a = _SCOPE.arena
    if a is None or not (recording or torch.is_grad_enabled() or _in_backward()):
        return torch.zeros(shape, dtype=dtype, device=device)
    return a.zeros(shape, dtype, device)


def _gn_bwd(dy, x, A, Bc, S, mr, gamma, beta, G, act, add, dx, dgamma, dbeta, dx_colsum, B, V, C, s, reduce=True):
    """og_affine_act_bwd_reduce (unless S already holds it) + og_gn_act_bwd on bf16 [B, V, C] tensors (the ResidualBlock's
    GroupNorm(1, C) / SiLU backward, genie/module/video.py:607-629)."""
    if reduce:
        _lib.call('og_affine_act_bwd_reduce', dy.data_ptr(), x.data_ptr(), A.data_ptr(), Bc.data_ptr(), act, S.data_ptr(),
                  B, V, C, *_scratch(dy), s)
    _lib.call('og_gn_act_bwd', dy.data_ptr(), x.data_ptr(), A.data_ptr(), Bc.data_ptr(), S.data_ptr(), mr.data_ptr(),
              gamma.data_ptr(), beta.data_ptr(), None, G, act, _ptr(add), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(),
              None, None, _ptr(dx_colsum), B, V, C, *_scratch(dy), s)


def _scratch(t: Tensor):
    """(pointer, bytes) of the current step scope's reduction scratch on t's device, for the C-ABI workspace arguments."""
    buf = _SCOPE.scratch(t.device)
    return buf.data_ptr(), buf.numel()


def _workspace(dev, nbytes: int):
    """Reusable fp32 scratch for split-K convolutions (small T*H*W, deep K). One buffer per device and step scope;
    every use is stream-ordered (partial-sum slabs -> finish pass inside one og_conv3d_* call)."""
    return _SCOPE.workspace(dev, nbytes)


# Optional per-launch timing of the tensor-core kernels (bench.py's roofline): when PROFILE is a list, every
# conv launch appends (kind, flops, start_event, end_event). CUDA events on the launching stream; no syncs.
PROFILE = None


def _conv_call(kind: str, flops: float, name: str, *args):
    if PROFILE is None:
        return _lib.call(name, *args)
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.call(name, *args)
    e1.record()
    PROFILE.append((kind, flops, e0, e1, tuple(a for a in args if isinstance(a, int) and a < (1 << 20))))


def _ptr(t: Optional[Tensor]):
    return None if t is None else t.data_ptr()


def _require_cuda(t: Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f'open_genie_b200: {what} must be a CUDA tensor — this package has no CPU path '
                           f'(the CPU restatement lives in oracle/ and is test infrastructure only)')


def empty_internal(B: int, C: int, T: int, H: int, W: int, dtype=bf16, device='cuda') -> Tensor:
    """Logical (B,C,T,H,W), physical NDHWC."""
    return torch.empty((B, T, H, W, C), dtype=dtype, device=device).permute(0, 4, 1, 2, 3)


def is_internal(x: Tensor) -> bool:
    return x.dim() == 5 and x.permute(0, 2, 3, 4, 1).is_contiguous()


def to_internal(x: Tensor, dtype=bf16) -> Tensor:
    """Reference-format tensor (any layout / float dtype) -> internal format of `dtype` (no autograd)."""
    _require_cuda(x, 'input')
    if x.dim() != 5:
        raise ValueError(f'expected a 5-D (B,C,T,H,W) tensor, got shape {tuple(x.shape)}')
    if is_internal(x) and x.dtype == dtype:
        return x
    B, C, T, H, W = x.shape
    if is_internal(x):  # only the dtype differs: row copy with cast
        y = empty_internal(B, C, T, H, W, dtype, x.device)
        if dtype == bf16:
            _lib.call('og_copy_rows_to_bf16', x.data_ptr(), int(x.dtype == f32), C, y.data_ptr(), C, B * T * H * W, C,
                      _stream())
            return y
        return x.permute(0, 2, 3, 4, 1).to(dtype).permute(0, 4, 1, 2, 3)
    xs = x.detach()
    if xs.dtype != f32 or not xs.is_contiguous():
        xs = xs.to(f32).contiguous()
    y = empty_internal(B, C, T, H, W, dtype, x.device)
    _lib.call('og_ncdhw_f32_to_ndhwc', xs.data_ptr(), y.data_ptr(), int(dtype == f32), B, C, T * H * W, _stream())
    return y


def to_reference(x: Tensor) -> Tensor:
    """Internal-format tensor -> contiguous NCDHW fp32 (what the reference's public methods return)."""
    if not is_internal(x) or x.dtype not in (bf16, f32):
        return x.float().contiguous()
    B, C, T, H, W = x.shape
    y = torch.empty((B, C, T, H, W), dtype=f32, device=x.device)
    _lib.call('og_ndhwc_to_ncdhw_f32', x.data_ptr(), int(x.dtype == f32), y.data_ptr(), B, C, T * H * W, _stream())
    return y


def _padded_ld(t: Tensor) -> int:
    """Row pitch if `t` is a channel-slice [:, :C] of a wider internal bf16 tensor (as produced by
    og_mse_bwd / og_lfq_bwd, whose pad channels are written as zeros), else 0."""
    if t.dim() != 5 or t.dtype != bf16 or t.stride(1) != 1:
        return 0
    B, C, T, H, W = t.shape
    cp = t.stride(4)
    if cp >= C and t.stride(3) == W * cp and t.stride(2) == H * W * cp and t.stride(0) == T * H * W * cp:
        return cp
    return 0


def _as_bf16_rows(t: Tensor, C: int, cpad: int) -> Tensor:
    """Any gradient tensor of logical (B,C,T,H,W) -> bf16 internal rows [B*V][cpad] (zero padded)."""
    if cpad != C and _padded_ld(t) == cpad:
        return t                      # already a zero-padded row buffer: use its storage in place
    if not is_internal(t):
        t = to_internal(t, bf16)
    if t.dtype == bf16 and cpad == C:
        return t
    B, _, T, H, W = t.shape
    y = empty_internal(B, cpad, T, H, W, bf16, t.device)
    if t.dtype not in (bf16, f32):
        t = t.float()
    _lib.call('og_pad_channels', t.data_ptr(), int(t.dtype == f32), y.data_ptr(), B * T * H * W, C, cpad, _stream())
    return y


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


# ------------------------------------------------------------------------------------------------
# convolution
# ------------------------------------------------------------------------------------------------
class ConvGeom:
    """Static description of one conv layer (kernel, stride, causal/symmetric padding)."""

    def __init__(self, cin, cout, kernel, stride=(1, 1, 1), pad_t_front=None, causal=True):
        self.cin, self.cout = cin, cout
        self.kt, self.kh, self.kw = kernel
        self.st, self.sh, self.sw = stride
        self.ph, self.pw = (self.kh - 1) // 2, (self.kw - 1) // 2
        if pad_t_front is None:
            # CausalConv3d: (kt-1)*dil + (1 - stride_t)  (genie/module/video.py:155); symmetric conv: (kt-1)//2
            pad_t_front = (self.kt - 1) + (1 - self.st) if causal else (self.kt - 1) // 2
        self.pt = pad_t_front
        self.causal = causal
        self.ntaps = self.kt * self.kh * self.kw
        self.strided = stride != (1, 1, 1)
        # Every convolution is an implicit GEMM: stride 1 (`direct`) or strided (strided TMA boxes forward / weight
        # gradient, residue-class decomposition for the data gradient). A k-block of the kernels is 64 channels of one
        # tap, so an input with Cin not in 64Z (the 3- and 18-channel stem convolutions) is zero-padded to `cin_pad`
        # channels (a pass over a 3-channel tensor) and its packed weights likewise — for Cin = 3 that costs ~0.3 ms of
        # extra tensor-core time per training step and replaces a 134 MB im2col buffer + its two passes.
        self.cin_pad = _round_up(cin, 64)
        self.padded = self.cin_pad != cin
        self.direct = not self.strided
        self.strided_implicit = self.strided
        self.k_main = self.ntaps * cin                      # algorithmic reduction length (FLOP accounting)
        self.kpad = self.ntaps * self.cin_pad
        if self.strided and not causal:
            raise NotImplementedError('strided convolutions implement CausalConv3d geometry only')

    def out_dims(self, T, H, W):
        if self.direct:
            return T, H, W
        padded = (T + self.pt, H + 2 * self.ph, W + 2 * self.pw)
        if any(p < k for p, k in zip(padded, (self.kt, self.kh, self.kw))):
            # F.conv3d raises here too; the kernels reject such a shape rather than compute an output for it
            raise ValueError(f'strided conv: padded input {padded} (T,H,W = {(T, H, W)}) is smaller than the kernel '
                             f'{(self.kt, self.kh, self.kw)}')
        return ((T + self.pt - self.kt) // self.st + 1, (H + 2 * self.ph - self.kh) // self.sh + 1,
                (W + 2 * self.pw - self.kw) // self.sw + 1)


def pack_weight(weight: Tensor, dst: Tensor, col_off: int, cin_pad: int = 0):
    """fp32 (Cout,Cin,kt,kh,kw) parameter (channels_last_3d memory = [Cout][tap][Cin]) -> bf16 segment of the
    packed operand matrix dst[Cout][ld] starting at column col_off. With cin_pad > Cin every tap's Cin channels land at
    a pitch of cin_pad (the pad columns of `dst` stay zero): dst must then be exactly [Cout][ntaps*cin_pad]."""
    w = weight.detach()
    cout, cin = w.shape[0], w.shape[1]
    k = w.numel() // cout
    if not w.permute(0, 2, 3, 4, 1).is_contiguous():
        w = w.permute(0, 2, 3, 4, 1).contiguous()
    if cin_pad and cin_pad != cin:
        assert col_off == 0 and dst.shape[1] == (k // cin) * cin_pad
        _lib.call('og_copy_rows_to_bf16', w.data_ptr(), 1, cin, dst.data_ptr(), cin_pad, cout * (k // cin), cin, _stream())
        return
    _lib.call('og_copy_rows_to_bf16', w.data_ptr(), 1, k, dst.data_ptr() + 2 * col_off, dst.shape[1], cout, k, _stream())


def _pad_input_channels(xi: Tensor, cpad: int) -> Tensor:
    """internal bf16 (B,C,T,H,W) -> (B,cpad,T,H,W) with zero channels appended (narrow-Cin stem convolutions)."""
    B, C, T, H, W = xi.shape
    y = empty_internal(B, cpad, T, H, W, bf16, xi.device)
    _lib.call('og_pad_channels', xi.data_ptr(), 0, y.data_ptr(), B * T * H * W, C, cpad, _stream())
    return y


class _Conv3dFn(torch.autograd.Function):
    """y = conv(x; w, b) [+ conv1x1(x2; w2, b2)]   — og_conv3d_fwd / dgrad / wgrad, or their strided forms."""

    @staticmethod
    def forward(ctx, x, weight, bias, x2, weight2, bias2, packed, geom: ConvGeom, out_f32: bool, residual=None):
        _require_cuda(x, 'conv input')
        B, C, T, H, W = x.shape
        assert C == geom.cin, f'conv: expected {geom.cin} input channels, got {C}'
        s = _stream()
        xi = to_internal(x, bf16)
        if geom.padded:
            assert x2 is None, 'a narrow-Cin convolution cannot carry a fused shortcut'
            xi = _pad_input_channels(xi, geom.cin_pad)
        Cp = geom.cin_pad                      # channel count the kernels see
        To, Ho, Wo = geom.out_dims(T, H, W)
        y = empty_internal(B, geom.cout, To, Ho, Wo, f32 if out_f32 else bf16, x.device)
        ldw = packed.shape[1]
        ws = _workspace(x.device, B * To * Ho * Wo * geom.cout * 4)
        x2i = None
        resi = None
        if residual is not None:     # out = conv(x) + residual, added in fp32 inside the GEMM epilogue (stride-1 convs)
            assert geom.direct and not out_f32, 'the fused residual add needs a stride-1 convolution with a bf16 output'
            resi = to_internal(residual, bf16)
            assert tuple(resi.shape) == (B, geom.cout, To, Ho, Wo), 'residual must have the shape of the output'
        if geom.direct:
            c1 = 0
            if x2 is not None:
                x2i = to_internal(x2, bf16)
                c1 = x2i.shape[1]
            _conv_call('fwd', 2.0 * B * T * H * W * geom.cout * (geom.k_main + c1),
                       'og_conv3d_fwd', xi.data_ptr(), Cp, geom.kt, geom.kh, geom.kw, geom.pt, geom.ph, geom.pw,
                      _ptr(x2i), c1, packed.data_ptr(), ldw, _ptr(bias), _ptr(bias2), _ptr(resi), y.data_ptr(), int(out_f32),
                      B, T, H, W, geom.cout, ws.data_ptr(), ws.numel(), None, s)
        else:
            assert x2 is None
            _conv_call('fwd', 2.0 * B * To * Ho * Wo * geom.cout * geom.k_main,
                       'og_conv3d_strided_fwd', xi.data_ptr(), Cp, geom.kt, geom.kh, geom.kw, geom.st, geom.sh, geom.sw,
                       geom.pt, geom.ph, geom.pw, packed.data_ptr(), ldw, _ptr(bias), y.data_ptr(), int(out_f32), B, T, H,
                       W, geom.cout, s)
        ctx.geom = geom
        ctx.in_shape = (B, C, T, H, W)
        ctx.has_bias = (bias is not None, bias2 is not None)
        ctx.has_residual = residual is not None
        ctx.w_shapes = (weight.shape, None if weight2 is None else weight2.shape)
        ctx.save_for_backward(xi, x2i, packed)
        return y

    @staticmethod
    def backward(ctx, dy):
        geom: ConvGeom = ctx.geom
        xs, x2i, packed = ctx.saved_tensors
        B, C, T, H, W = ctx.in_shape
        To, Ho, Wo = geom.out_dims(T, H, W)
        s = _stream()
        ldw = packed.shape[1]
        cout = geom.cout
        cpad = _round_up(cout, 64)
        dyb = _as_bf16_rows(dy, cout, cpad)          # [B,To,Ho,Wo,cpad] bf16
        need = ctx.needs_input_grad
        dx = dw = db = dx2 = dw2 = db2 = None
        dev = dy.device
        ws = _workspace(dev, B * T * H * W * max(C, 64) * 4)

        want_db = (ctx.has_bias[0] and need[2]) or (ctx.has_bias[1] and need[5])
        dbs = _zeros(cout, f32, dev) if want_db else None
        fused_db = [False]

        def wgrad(xin, cin, kt, kh, kw, pt, ph, pw, shape5, dims):
            """fp32 gradient with the parameter's channels_last_3d memory: [cout][tap][cin]. The first weight gradient of
            this backward also produces the bias gradient (column sums of dy) when one is wanted."""
            rows = cpad if cpad != cout else cout
            g = _zeros((rows, kt * kh * kw * cin), f32, dev)
            real_cin = C if (geom.padded and cin == geom.cin_pad) else cin      # algorithmic FLOPs: no padding counted
            fl = 2.0 * dims[0] * dims[1] * dims[2] * dims[3] * cout * min(real_cin, geom.k_main) * kt * kh * kw
            if want_db and not fused_db[0]:
                fused_db[0] = True
                _conv_call('wgrad', fl, 'og_conv3d_wgrad_bias', dyb.data_ptr(), cpad, xin.data_ptr(), cin, g.data_ptr(),
                           g.shape[1], kt, kh, kw, pt, ph, pw, dims[0], dims[1], dims[2], dims[3], dbs.data_ptr(), cout,
                           *_scratch(dyb), s)
            else:
                _conv_call('wgrad', fl, 'og_conv3d_wgrad', dyb.data_ptr(), cpad, xin.data_ptr(), cin, g.data_ptr(), g.shape[1],
                           kt, kh, kw, pt, ph, pw, dims[0], dims[1], dims[2], dims[3], *_scratch(dyb), s)
            return g[:cout]

        Cp = geom.cin_pad
        if geom.direct:
            if need[0]:
                dx = empty_internal(B, Cp, T, H, W, bf16, dev)
                _conv_call('dgrad', 2.0 * B * T * H * W * cout * geom.k_main,
                           'og_conv3d_dgrad', dyb.data_ptr(), cpad, cout, packed.data_ptr(), ldw, 0, geom.kt, geom.kh,
                           geom.kw, geom.pt, geom.ph, geom.pw, dx.data_ptr(), 0, B, T, H, W, Cp, ws.data_ptr(), ws.numel(),
                           s)
                if geom.padded:
                    dx = dx[:, :C]
            if need[1]:
                g = wgrad(xs, Cp, geom.kt, geom.kh, geom.kw, geom.pt, geom.ph, geom.pw, ctx.w_shapes[0], (B, T, H, W))
                dw = g.view(cout, geom.kt, geom.kh, geom.kw, Cp)[..., :C].permute(0, 4, 1, 2, 3)
            if x2i is not None:
                c1 = x2i.shape[1]
                if need[3]:
                    dx2 = empty_internal(B, c1, T, H, W, bf16, dev)
                    _conv_call('dgrad', 2.0 * B * T * H * W * cout * c1,
                               'og_conv3d_dgrad', dyb.data_ptr(), cpad, cout, packed.data_ptr(), ldw, geom.k_main,
                               1, 1, 1, 0, 0, 0, dx2.data_ptr(), 0, B, T, H, W, c1, ws.data_ptr(), ws.numel(), s)
                if need[4]:
                    g = wgrad(x2i, c1, 1, 1, 1, 0, 0, 0, ctx.w_shapes[1], (B, T, H, W))
                    dw2 = g.view(cout, 1, 1, 1, c1).permute(0, 4, 1, 2, 3)
        else:
            if need[0]:
                dx = empty_internal(B, Cp, T, H, W, bf16, dev)
                _conv_call('dgrad', 2.0 * B * To * Ho * Wo * cout * geom.k_main,
                           'og_conv3d_strided_dgrad', dyb.data_ptr(), cpad, cout, packed.data_ptr(), ldw, geom.kt, geom.kh,
                           geom.kw, geom.st, geom.sh, geom.sw, geom.pt, geom.ph, geom.pw, dx.data_ptr(), B, T, H, W, Cp, s)
                if geom.padded:
                    dx = dx[:, :C]
            if need[1]:
                rows = cpad if cpad != cout else cout
                g = _zeros((rows, geom.ntaps * Cp), f32, dev)
                _conv_call('wgrad', 2.0 * B * To * Ho * Wo * cout * geom.k_main,
                           'og_conv3d_strided_wgrad', dyb.data_ptr(), cpad, xs.data_ptr(), Cp, g.data_ptr(), g.shape[1],
                           geom.kt, geom.kh, geom.kw, geom.st, geom.sh, geom.sw, geom.pt, geom.ph, geom.pw, B, T, H, W,
                           *_scratch(dyb), s)
                dw = g[:cout].view(cout, geom.kt, geom.kh, geom.kw, Cp)[..., :C].permute(0, 4, 1, 2, 3)
        if want_db:
            if not fused_db[0]:
                _lib.call('og_colsum', dyb.data_ptr(), B * To * Ho * Wo, cout, cpad, dbs.data_ptr(), s)
            if ctx.has_bias[0] and need[2]:
                db = dbs
            if ctx.has_bias[1] and need[5]:
                db2 = dbs if db is None else dbs.clone()
        return dx, dw, db, dx2, dw2, db2, None, None, None, (dyb[:, :cout] if ctx.has_residual else None)


def conv3d(x, weight, bias, packed, geom, out_f32=False, x2=None, weight2=None, bias2=None, residual=None):
    return _Conv3dFn.apply(x, weight, bias, x2, weight2, bias2, packed, geom, out_f32, residual)


# ------------------------------------------------------------------------------------------------
# GroupNorm / AdaGN (+ SiLU)
# ------------------------------------------------------------------------------------------------
class _GroupNormActFn(torch.autograd.Function):
    """y = act(GN_G(x; gamma, beta) * cond_scale + cond_shift)"""

    @staticmethod
    def forward(ctx, x, gamma, beta, cond_scale, cond_shift, G: int, eps: float, act: int):
        _require_cuda(x, 'group_norm input')
        xi = to_internal(x, bf16)
        B, C, T, H, W = xi.shape
        V = T * H * W
        s = _stream()
        dev = xi.device
        sums = _zeros((B, G, 2), torch.float64, dev, any(ctx.needs_input_grad))
        _lib.call('og_gn_stats', xi.data_ptr(), B, V, C, G, sums.data_ptr(), s)
        A = torch.empty((B, C), dtype=f32, device=dev)
        Bc = torch.empty((B, C), dtype=f32, device=dev)
        mr = torch.empty((B, G, 2), dtype=f32, device=dev)
        cs = None if cond_scale is None else cond_scale.detach().to(f32).contiguous()
        csh = None if cond_shift is None else cond_shift.detach().to(f32).contiguous()
        y = empty_internal(B, C, T, H, W, bf16, dev)
        if (C // G) % 8 == 0:
            _lib.call('og_gn_act_fwd', xi.data_ptr(), sums.data_ptr(), _ptr(gamma), _ptr(beta), _ptr(cs), _ptr(csh), eps,
                      G, act, y.data_ptr(), A.data_ptr(), Bc.data_ptr(), mr.data_ptr(), B, V, C, s)
        else:
            _lib.call('og_gn_finalize', sums.data_ptr(), B, C, G, V, eps, _ptr(gamma), _ptr(beta), _ptr(cs), _ptr(csh),
                      A.data_ptr(), Bc.data_ptr(), mr.data_ptr(), s)
            _lib.call('og_affine_act_fwd', xi.data_ptr(), A.data_ptr(), Bc.data_ptr(), y.data_ptr(), B, V, C, act, s)
        ctx.cfg = (G, act, cond_scale is not None, cond_shift is not None)
        ctx.save_for_backward(xi, A, Bc, mr, gamma, beta, cs)
        return y

    @staticmethod
    def backward(ctx, dy):
        xi, A, Bc, mr, gamma, beta, cs = ctx.saved_tensors
        G, act, has_cs, has_csh = ctx.cfg
        B, C, T, H, W = xi.shape
        V = T * H * W
        s = _stream()
        dev = xi.device
        dyb = _as_bf16_rows(dy, C, C)
        S = _zeros((B, C, 2), f32, dev)
        _lib.call('og_affine_act_bwd_reduce', dyb.data_ptr(), xi.data_ptr(), A.data_ptr(), Bc.data_ptr(), act,
                  S.data_ptr(), B, V, C, *_scratch(dyb), s)
        dgamma = _zeros(C, f32, dev) if gamma is not None else None
        dbeta = _zeros(C, f32, dev) if beta is not None else None
        dcs = torch.empty((B, C), dtype=f32, device=dev) if has_cs else None
        dcsh = torch.empty((B, C), dtype=f32, device=dev) if has_csh else None
        dx = None
        if (C // G) % 8 == 0 and ctx.needs_input_grad[0]:
            dx = empty_internal(B, C, T, H, W, bf16, dev)
            _lib.call('og_gn_act_bwd', dyb.data_ptr(), xi.data_ptr(), A.data_ptr(), Bc.data_ptr(), S.data_ptr(),
                      mr.data_ptr(), _ptr(gamma), _ptr(beta), _ptr(cs), G, act, None, dx.data_ptr(), _ptr(dgamma),
                      _ptr(dbeta), _ptr(dcs), _ptr(dcsh), None, B, V, C, *_scratch(dyb), s)
            return dx, dgamma, dbeta, dcs, dcsh, None, None, None
        Q = torch.empty((B, C), dtype=f32, device=dev)
        R = torch.empty((B, C), dtype=f32, device=dev)
        _lib.call('og_gn_bwd_finalize', S.data_ptr(), mr.data_ptr(), _ptr(gamma), _ptr(beta), _ptr(cs), B, C, G, V,
                  Q.data_ptr(), R.data_ptr(), _ptr(dgamma), _ptr(dbeta), _ptr(dcs), _ptr(dcsh), s)
        if ctx.needs_input_grad[0]:
            dx = empty_internal(B, C, T, H, W, bf16, dev)
            _lib.call('og_affine_act_bwd_apply', dyb.data_ptr(), xi.data_ptr(), A.data_ptr(), Bc.data_ptr(),
                      Q.data_ptr(), R.data_ptr(), None, dx.data_ptr(), act, B, V, C, s)
        return dx, dgamma, dbeta, dcs, dcsh, None, None, None


ACT_CODES = {'none': 0, None: 0, 'silu': 1, 'swish': 1, 'leaky': 2, 'leaky_relu': 2, 'relu': 3}


def act_code(act) -> int:
    """Activation name -> kernel code (csrc/norm_act.cu): 0 identity, 1 SiLU, 2 LeakyReLU(0.01), 3 ReLU."""
    if isinstance(act, int):
        return act
    if act not in ACT_CODES:
        raise ValueError(f'unknown activation {act!r}')
    return ACT_CODES[act]


def group_norm_act(x, gamma, beta, num_groups, eps=1e-5, act='none', cond_scale=None, cond_shift=None):
    return _GroupNormActFn.apply(x, gamma, beta, cond_scale, cond_shift, num_groups, eps, act_code(act))


class _AdaGNCondFn(torch.autograd.Function):
    """(scale, shift) = (W_s cbar + b_s, W_a cbar + b_a), cbar = mean_{t,h,w}(cond) — AdaptiveGroupNorm.forward's
    conditioning path (genie/module/norm.py:58-66) in one launch each way (og_adagn_cond_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, cond, w_s, b_s, w_a, b_a):
        _require_cuda(cond, 'AdaGN condition')
        B, D = cond.shape[0], cond.shape[1]
        rows = cond.detach().movedim(1, -1)                       # (B, ..., D): free for channels-last conditions
        if rows.dtype != f32 or not rows.is_contiguous():
            rows = rows.to(f32).contiguous()
        V = rows.numel() // (B * D)
        C = w_s.shape[0]
        dev = cond.device
        cbar = torch.empty((B, D), dtype=f32, device=dev)
        scale = torch.empty((B, C), dtype=f32, device=dev)
        shift = torch.empty((B, C), dtype=f32, device=dev) if w_a is not None else None
        _lib.call('og_adagn_cond_fwd', rows.data_ptr(), B, V, D, w_s.data_ptr(), _ptr(b_s), _ptr(w_a), _ptr(b_a), C,
                  cbar.data_ptr(), scale.data_ptr(), _ptr(shift), _stream())
        ctx.cfg = (tuple(cond.shape), V, w_a is not None)
        ctx.save_for_backward(cbar, w_s, w_a)
        return scale, shift

    @staticmethod
    def backward(ctx, dscale, dshift):
        cbar, w_s, w_a = ctx.saved_tensors
        shape, V, has_shift = ctx.cfg
        B, D = shape[0], shape[1]
        C = w_s.shape[0]
        dev = cbar.device
        ds = dscale.detach().to(f32).contiguous()
        dh = dshift.detach().to(f32).contiguous() if (has_shift and dshift is not None) else None
        dws = torch.empty_like(w_s, dtype=f32)
        dbs = torch.empty((C,), dtype=f32, device=dev)
        dwa = torch.empty_like(w_a, dtype=f32) if has_shift else None
        dba = torch.empty((C,), dtype=f32, device=dev) if has_shift else None
        dcond = None
        if ctx.needs_input_grad[0]:
            dcond = torch.empty((B,) + tuple(shape[2:]) + (D,), dtype=f32, device=dev)
        _lib.call('og_adagn_cond_bwd', ds.data_ptr(), _ptr(dh), cbar.data_ptr(), w_s.data_ptr(), _ptr(w_a), B, V, D, C,
                  dws.data_ptr(), dbs.data_ptr(), _ptr(dwa), _ptr(dba), _ptr(dcond), _stream())
        return (dcond.movedim(-1, 1) if dcond is not None else None), dws, dbs, dwa, dba


def adagn_condition(cond, w_scale, b_scale, w_shift=None, b_shift=None):
    return _AdaGNCondFn.apply(cond, w_scale, b_scale, w_shift, b_shift)


class _ActFn(torch.autograd.Function):
    """Stand-alone activation y = act(scale * x): blueprint entry 'silu' (genie/tokenizer.py:79,167), the discriminators'
    nn.LeakyReLU() (discriminator.py:97), VGG's ReLU, and plain scaling (act = 0)."""

    @staticmethod
    def forward(ctx, x, act: int, scale: float):
        xi = to_internal(x, bf16)
        B, C, T, H, W = xi.shape
        dev = xi.device
        A = torch.full((B, C), float(scale), dtype=f32, device=dev)
        Bc = torch.zeros((B, C), dtype=f32, device=dev)
        y = empty_internal(B, C, T, H, W, bf16, dev)
        _lib.call('og_affine_act_fwd', xi.data_ptr(), A.data_ptr(), Bc.data_ptr(), y.data_ptr(), B, T * H * W, C, act,
                  _stream())
        ctx.act = act
        ctx.save_for_backward(xi, A, Bc)
        return y

    @staticmethod
    def backward(ctx, dy):
        xi, A, Bc = ctx.saved_tensors
        B, C, T, H, W = xi.shape
        dyb = _as_bf16_rows(dy, C, C)
        dx = empty_internal(B, C, T, H, W, bf16, xi.device)
        _lib.call('og_affine_act_bwd_apply', dyb.data_ptr(), xi.data_ptr(), A.data_ptr(), Bc.data_ptr(), None, None,
                  None, dx.data_ptr(), ctx.act, B, T * H * W, C, _stream())
        return dx, None, None


def silu(x):
    return _ActFn.apply(x, 1, 1.0)


def activation(x, act='none', scale: float = 1.0):
    """y = act(scale * x) on an internal-format (C % 8 == 0) tensor."""
    return _ActFn.apply(x, act_code(act), float(scale))


# ------------------------------------------------------------------------------------------------
# pixel shuffle (depth -> space-time)
# ------------------------------------------------------------------------------------------------
class _PixelShuffleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p: int, q: int, r: int):
        xi = to_internal(x, bf16)
        B, CC, T, H, W = xi.shape
        c = CC // (p * q * r)
        y = empty_internal(B, c, T * p, H * q, W * r, bf16, xi.device)
        _lib.call('og_pixel_shuffle3d', xi.data_ptr(), y.data_ptr(), 0, B, T, H, W, c, p, q, r, _stream())
        ctx.cfg = (B, CC, T, H, W, c, p, q, r)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, CC, T, H, W, c, p, q, r = ctx.cfg
        dyb = _as_bf16_rows(dy, c, c)
        dx = empty_internal(B, CC, T, H, W, bf16, dy.device)
        _lib.call('og_pixel_shuffle3d', dx.data_ptr(), dyb.data_ptr(), 1, B, T, H, W, c, p, q, r, _stream())
        return dx, None, None, None


def pixel_shuffle3d(x, p, q, r):
    return _PixelShuffleFn.apply(x, p, q, r)


class _SpaceToDepthFn(torch.autograd.Function):
    """'b c (t p) (h q) (w r) -> b (c p q r) t h w' — the inverse shuffle, forward op of SpaceDownsample
    (genie/module/image.py:92-95 with p = 1). Same kernel as _PixelShuffleFn run in its other direction."""

    @staticmethod
    def forward(ctx, x, p: int, q: int, r: int):
        xi = to_internal(x, bf16)
        B, c, Tp, Hq, Wr = xi.shape
        assert Tp % p == 0 and Hq % q == 0 and Wr % r == 0, 'space_to_depth: extents must divide by the factors'
        T, H, W = Tp // p, Hq // q, Wr // r
        y = empty_internal(B, c * p * q * r, T, H, W, bf16, xi.device)
        _lib.call('og_pixel_shuffle3d', y.data_ptr(), xi.data_ptr(), 1, B, T, H, W, c, p, q, r, _stream())
        ctx.cfg = (B, c, T, H, W, p, q, r)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, c, T, H, W, p, q, r = ctx.cfg
        dyb = _as_bf16_rows(dy, c * p * q * r, c * p * q * r)
        dx = empty_internal(B, c, T * p, H * q, W * r, bf16, dy.device)
        _lib.call('og_pixel_shuffle3d', dyb.data_ptr(), dx.data_ptr(), 0, B, T, H, W, c, p, q, r, _stream())
        return dx, None, None, None


def space_to_depth3d(x, p, q, r):
    return _SpaceToDepthFn.apply(x, p, q, r)


# ------------------------------------------------------------------------------------------------
# blur pooling
# ------------------------------------------------------------------------------------------------
class _BlurPoolFn(torch.autograd.Function):
    """BlurPooling3d with `groups` groups: og_blurpool3d at groups == 1, og_blurpool3d_grouped otherwise."""

    @staticmethod
    def forward(ctx, x, k: int, stride, cout: int, groups: int = 1):
        xi = to_internal(x, bf16)
        B, C, T, H, W = xi.shape
        st, sh, sw = stride
        pad = (k - 1) // 2
        To, Ho, Wo = (T + 2 * pad - k) // st + 1, (H + 2 * pad - k) // sh + 1, (W + 2 * pad - k) // sw + 1
        y = empty_internal(B, cout, To, Ho, Wo, bf16, xi.device)
        scratch = torch.empty(B * T * H * W * groups, dtype=f32, device=xi.device)
        if groups == 1:
            _lib.call('og_blurpool3d', xi.data_ptr(), y.data_ptr(), scratch.data_ptr(), 0, B, T, H, W, C, cout, k, st, sh,
                      sw, _stream())
        else:
            _lib.call('og_blurpool3d_grouped', xi.data_ptr(), y.data_ptr(), scratch.data_ptr(), 0, B, T, H, W, C, cout,
                      groups, k, st, sh, sw, _stream())
        ctx.cfg = (B, C, T, H, W, cout, k, st, sh, sw, To, Ho, Wo, groups)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, C, T, H, W, cout, k, st, sh, sw, To, Ho, Wo, groups = ctx.cfg
        dyb = _as_bf16_rows(dy, cout, cout)
        dx = empty_internal(B, C, T, H, W, bf16, dy.device)
        scratch = torch.empty(B * To * Ho * Wo * groups, dtype=f32, device=dy.device)
        if groups == 1:
            _lib.call('og_blurpool3d', dyb.data_ptr(), dx.data_ptr(), scratch.data_ptr(), 1, B, T, H, W, C, cout, k, st,
                      sh, sw, _stream())
        else:
            _lib.call('og_blurpool3d_grouped', dyb.data_ptr(), dx.data_ptr(), scratch.data_ptr(), 1, B, T, H, W, C, cout,
                      groups, k, st, sh, sw, _stream())
        return dx, None, None, None, None


def blurpool3d(x, k, stride, cout, groups=1):
    return _BlurPoolFn.apply(x, k, tuple(stride), cout, groups)


# ------------------------------------------------------------------------------------------------
# mse loss between an internal fp32 reconstruction and the reference-format target
# ------------------------------------------------------------------------------------------------
class _MseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rec, target):
        assert is_internal(rec) and rec.dtype == f32, 'mse: reconstruction must be internal fp32'
        B, C, T, H, W = rec.shape
        tgt = target.detach()
        if tgt.dtype != f32 or not tgt.is_contiguous():
            tgt = tgt.to(f32).contiguous()
        acc = torch.zeros((), dtype=f32, device=rec.device)
        _lib.call('og_mse_fwd', rec.data_ptr(), tgt.data_ptr(), B, C, T * H * W, acc.data_ptr(), _stream())
        ctx.save_for_backward(rec, tgt)
        return acc / float(rec.numel())

    @staticmethod
    def backward(ctx, g):
        rec, tgt = ctx.saved_tensors
        B, C, T, H, W = rec.shape
        cpad = _round_up(C, 64)
        gs = g.detach().to(f32).contiguous()
        drec = empty_internal(B, cpad, T, H, W, bf16, rec.device)
        _lib.call('og_mse_bwd', rec.data_ptr(), tgt.data_ptr(), gs.data_ptr(), B, C, cpad, T * H * W, drec.data_ptr(),
                  _stream())
        return drec[:, :C], None


def mse_loss(rec, target):
    return _MseFn.apply(rec, target)


# ------------------------------------------------------------------------------------------------
# Lookup-free quantisation
# ------------------------------------------------------------------------------------------------
class _LfqFn(torch.autograd.Function):
    """x: fp32 [ntok, C*D] -> (out fp32 [ntok, C*D], idx int64 [ntok] (C = 1) or [ntok, C], loss scalar or None).
    C = 1 runs og_lfq_fwd / og_lfq_bwd; C > 1 the multi-codebook entry points."""

    @staticmethod
    def forward(ctx, x, D, beta, training, w_commit, w_entropy, w_div, C):
        _require_cuda(x, 'lfq input')
        xs = x.detach()
        if xs.dtype != f32 or not xs.is_contiguous():
            xs = xs.to(f32).contiguous()
        ntok = xs.shape[0]
        dev = xs.device
        out = torch.empty((ntok, C * D), dtype=f32, device=dev)
        idx = torch.empty((ntok,) if C == 1 else (ntok, C), dtype=torch.int64, device=dev)
        loss = torch.zeros((), dtype=f32, device=dev)
        ws = None
        if training:
            if C == 1:
                nbytes = _lib.load().og_lfq_workspace_bytes(ntok, D)
            else:
                nbytes = _lib.load().og_lfq_multi_workspace_bytes(ntok, D, C)
            if nbytes == 0:
                raise RuntimeError(f'lfq: codebook_dim={D}, n_codebook={C} is outside the supported range '
                                   f'(codebook_dim in [1, 20], n_codebook in [1, 65535])')
            ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        if C == 1:
            _lib.call('og_lfq_fwd', xs.data_ptr(), xs.shape[1], ntok, D, beta, int(training), w_commit, w_entropy,
                      w_div, out.data_ptr(), None, 0, idx.data_ptr(), loss.data_ptr(), _ptr(ws), _stream())
        else:
            _lib.call('og_lfq_multi_fwd', xs.data_ptr(), xs.shape[1], ntok, D, C, beta, int(training), w_commit,
                      w_entropy, w_div, out.data_ptr(), None, 0, idx.data_ptr(), loss.data_ptr(), _ptr(ws), _stream())
        ctx.cfg = (D, beta, w_commit, w_entropy, training, C)
        ctx.save_for_backward(xs, ws)
        ctx.mark_non_differentiable(idx)
        return out, idx, loss

    @staticmethod
    def backward(ctx, dout, _didx, dloss):
        D, beta, w_commit, w_entropy, training, C = ctx.cfg
        xs, ws = ctx.saved_tensors
        if not training:
            return (None,) * 8     # eval: code = sign(x) has no gradient path (quantization.py:101)
        ntok = xs.shape[0]
        dx = torch.empty((ntok, C * D), dtype=f32, device=xs.device)
        do = None if dout is None else dout.detach().to(f32).contiguous()
        gl = dloss.detach().to(f32).contiguous() if dloss is not None else torch.zeros((), device=xs.device)
        if C == 1:
            _lib.call('og_lfq_bwd', xs.data_ptr(), xs.shape[1], ntok, D, beta, w_commit, w_entropy, gl.data_ptr(),
                      _ptr(do), D, dx.data_ptr(), None, D, ws.data_ptr(), _stream())
        else:
            _lib.call('og_lfq_multi_bwd', xs.data_ptr(), xs.shape[1], ntok, D, C, beta, w_commit, w_entropy,
                      gl.data_ptr(), _ptr(do), C * D, dx.data_ptr(), None, C * D, ws.data_ptr(), _stream())
        return dx, None, None, None, None, None, None, None


def lfq(x2d, D, beta, training, w_commit, w_entropy, w_div, n_codebook=1):
    """Lookup-free quantisation of x2d [ntok, n_codebook * D] (quantization.py:77-133): n_codebook independent D-bit
    codes per token, their straight-through output, indices ([ntok], or [ntok, n_codebook] when n_codebook > 1) and,
    in training, the entropy + commitment loss."""
    return _LfqFn.apply(x2d, D, float(beta), bool(training), float(w_commit), float(w_entropy), float(w_div),
                        int(n_codebook))


# ------------------------------------------------------------------------------------------------
# factored space-time attention (tensors here are plain contiguous (B, T, H, W, C) bf16 == NDHWC rows)
# ------------------------------------------------------------------------------------------------
def _rows_bf16(x: Tensor) -> Tensor:
    """(B,T,H,W,C) contiguous bf16 view of a tensor in either logical layout (no copy when already internal)."""
    if x.dtype != bf16 or not x.is_contiguous():
        x = x.to(bf16).contiguous()
    return x


def _rope_table(freq: Tensor, npos: int) -> Optional[Tensor]:
    """fp32 (npos, C/2, 2) table of (cos, sin)(pos * freq) for the fused RoPE+LayerNorm passes. Cached ON the frequency
    tensor object (per sequence length; rebuilt if the tensor is modified in place), so it lives and dies with the module's
    `freq` parameter. Never built while a CUDA graph is being captured: a captured step uses the tables its warm-up steps
    created, or none (the passes then evaluate sincosf per element — same values)."""
    cache = getattr(freq, '_og_rope_tables', None)
    if cache is None or cache[0] != (freq.data_ptr(), freq._version):
        cache = ((freq.data_ptr(), freq._version), {})
        try:
            freq._og_rope_tables = cache
        except Exception:
            return None
    t = cache[1].get(int(npos))
    if t is None:
        if torch.cuda.is_current_stream_capturing():
            return None
        C = 2 * freq.numel()
        t = torch.empty((npos, C // 2, 2), dtype=f32, device=freq.device)
        _lib.call('og_rope_table', freq.detach().float().contiguous().data_ptr(), int(npos), C, t.data_ptr(), _stream())
        cache[1][int(npos)] = t
    return t


def _ln_rows_fwd(x: Tensor, freq: Optional[Tensor], gamma: Tensor, beta: Tensor, eps: float, q: Tensor, rows: int,
                 C: int, pos_div: int, pos_mod: int, s) -> None:
    """q = LayerNorm(RoPE(x)) with the rotary frequencies `freq`, or q = LayerNorm(x) when freq is None (embed=False)."""
    if freq is None:
        _lib.call('og_ln_rows_fwd', x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps, q.data_ptr(), rows, C, s)
    else:
        _lib.call('og_rope_ln_fwd', x.data_ptr(), freq.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps,
                  q.data_ptr(), rows, C, pos_div, pos_mod, _ptr(_rope_table(freq, pos_mod)), s)


def _ln_rows_bwd(x: Tensor, freq: Optional[Tensor], gamma: Tensor, eps: float, g0: Tensor, g1, g2, add: Tensor,
                 dx: Tensor, dgamma: Tensor, dbeta: Tensor, rows: int, C: int, pos_div: int, pos_mod: int, s) -> None:
    """The backward pass of _ln_rows_fwd for the gradient g0 + g1 + g2 (g1, g2 may be None), plus `add`."""
    if freq is None:
        _lib.call('og_ln_rows_bwd', x.data_ptr(), gamma.data_ptr(), eps, g0.data_ptr(), _ptr(g1), _ptr(g2),
                  add.data_ptr(), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), rows, C, s)
    else:
        _lib.call('og_rope_ln_bwd', x.data_ptr(), freq.data_ptr(), gamma.data_ptr(), eps, g0.data_ptr(), _ptr(g1),
                  _ptr(g2), add.data_ptr(), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), rows, C, pos_div,
                  pos_mod, _ptr(_rope_table(freq, pos_mod)), s)


def _dropout_seed(device) -> Tensor:
    """The seed of one attention call with dropout: one int64 (read by the kernels as a uint64) drawn from the current
    CUDA generator on the device, so torch.manual_seed governs the masks and a CUDA-graph replay, whose capture
    registers the generator, draws a fresh seed. The forward pass saves it for the backward pass."""
    return torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=device)


class _SpaceAttnFn(torch.autograd.Function):
    """y = SDPA(q, q, q; scale, dropout_p) + x with q = LayerNorm(RoPE2d(x)), sequences = frames (H*W tokens).
    SpatialAttention.forward + the residual of SpaceTimeAttention.forward (attention.py:279-307, 470).
    freq = None (embed=False) gives q = LayerNorm(x), through og_ln_rows_fwd / bwd.
    dropout > 0 runs og_flash_attn_dropout_fwd / bwd with a seed from _dropout_seed; 0 runs og_flash_attn_fwd / bwd.
    causal (SpatialAttention(causal=True): SDPA is_causal=True over the H*W tokens in raster order) runs
    og_flash_attn_causal_fwd / bwd at every dropout, with a seed only when dropout > 0."""

    @staticmethod
    def forward(ctx, x, freq, gamma, beta, n_head: int, scale: float, eps: float, dropout: float,
                causal: bool = False):
        _require_cuda(x, 'attention input')
        x = _rows_bf16(x)
        B, T, H, W, C = x.shape
        rows, S = B * T * H * W, H * W
        s = _stream()
        q = torch.empty_like(x)
        _ln_rows_fwd(x, freq, gamma, beta, eps, q, rows, C, 1, S, s)
        y, o = torch.empty_like(x), torch.empty_like(x)
        lse = torch.empty((B * T, n_head, S), dtype=f32, device=x.device)
        seed = _dropout_seed(x.device) if dropout > 0 else None
        if causal:   # the S (S + 1) / 2 scores with key <= query
            _conv_call('attn_fwd', 2.0 * B * T * S * (S + 1) * C, 'og_flash_attn_causal_fwd', q.data_ptr(), q.data_ptr(),
                       q.data_ptr(), o.data_ptr(), x.data_ptr(), y.data_ptr(), lse.data_ptr(), B * T, S, C, n_head,
                       scale, dropout, _ptr(seed), s)
        elif dropout > 0:
            _conv_call('attn_fwd', 4.0 * B * T * S * S * C, 'og_flash_attn_dropout_fwd', q.data_ptr(), q.data_ptr(),
                       q.data_ptr(), o.data_ptr(), x.data_ptr(), y.data_ptr(), lse.data_ptr(), B * T, S, C, n_head,
                       scale, dropout, seed.data_ptr(), s)
        else:
            _conv_call('attn_fwd', 4.0 * B * T * S * S * C, 'og_flash_attn_fwd', q.data_ptr(), q.data_ptr(),
                       q.data_ptr(), o.data_ptr(), x.data_ptr(), y.data_ptr(), lse.data_ptr(), B * T, S, C, n_head,
                       scale, s)
        ctx.cfg = (n_head, scale, eps, dropout, causal)
        ctx.save_for_backward(x, q, o, lse, freq, gamma, seed)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, q, o, lse, freq, gamma, seed = ctx.saved_tensors
        n_head, scale, eps, dropout, causal = ctx.cfg
        B, T, H, W, C = x.shape
        rows, S = B * T * H * W, H * W
        s = _stream()
        dy = _rows_bf16(dy)
        dq, dk, dv = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
        delta = torch.empty_like(lse)
        if causal:
            _conv_call('attn_bwd', 5.0 * B * T * S * (S + 1) * C, 'og_flash_attn_causal_bwd', q.data_ptr(), q.data_ptr(),
                       q.data_ptr(), o.data_ptr(), dy.data_ptr(), lse.data_ptr(), delta.data_ptr(), dq.data_ptr(),
                       dk.data_ptr(), dv.data_ptr(), B * T, S, C, n_head, scale, dropout, _ptr(seed), s)
        elif dropout > 0:
            _conv_call('attn_bwd', 10.0 * B * T * S * S * C, 'og_flash_attn_dropout_bwd', q.data_ptr(), q.data_ptr(),
                       q.data_ptr(), o.data_ptr(), dy.data_ptr(), lse.data_ptr(), delta.data_ptr(), dq.data_ptr(),
                       dk.data_ptr(), dv.data_ptr(), B * T, S, C, n_head, scale, dropout, seed.data_ptr(), s)
        else:
            _conv_call('attn_bwd', 10.0 * B * T * S * S * C, 'og_flash_attn_bwd', q.data_ptr(), q.data_ptr(),
                       q.data_ptr(), o.data_ptr(), dy.data_ptr(), lse.data_ptr(), delta.data_ptr(), dq.data_ptr(),
                       dk.data_ptr(), dv.data_ptr(), B * T, S, C, n_head, scale, s)
        dx = torch.empty_like(x)
        dgamma = _zeros(C, f32, x.device)
        dbeta = _zeros(C, f32, x.device)
        _ln_rows_bwd(x, freq, gamma, eps, dq, dk, dv, dy, dx, dgamma, dbeta, rows, C, 1, S, s)
        return dx, None, dgamma, dbeta, None, None, None, None, None


# Longest clip of the per-pixel temporal kernels (og_temporal_attn_fwd / bwd); longer ones take the tiled kernels.
_TIME_ATTN_SHORT_T = 32


def _time_attn_tiled(T: int, C: int, n_head: int, dropout: float = 0.0) -> bool:
    """Whether temporal attention runs on the tiled kernels (og_temporal_attn_long_fwd / bwd): clips longer than
    _TIME_ATTN_SHORT_T, and every clip at d_head = 128 or 16. With dropout every clip does: only the tiled kernels
    drop (og_temporal_attn_long_dropout_fwd / bwd), and they take any T >= 1. The per-pixel kernels do not take 128 (a lane would hold
    2 x 128 fp32 values). At 16 they would not be faster: timed at T = 16, B = 8, 256 pixels, 16 heads of 16 (H100
    80GB HBM3, 700 W), the per-pixel kernels instantiated at 16 took 0.124 + 0.333 ms (fwd + bwd) against the tiled
    kernels' 0.123 + 0.334 ms, and 0.111 + 0.287 ms against 0.123 + 0.252 ms with broadcast K / V."""
    return dropout > 0 or T > _TIME_ATTN_SHORT_T or C == 128 * n_head or C == 16 * n_head


class _TimeAttnFn(torch.autograd.Function):
    """y = SDPA_causal(q, k, v; scale, dropout_p) + x over t for every pixel; q = LayerNorm(RoPE1d(x)); k = v = q, or
    the projected latent-action conditioning (B, T, C) shared by all pixels (attention.py:347-371, 471).
    freq = None (embed=False) gives q = LayerNorm(x), through og_ln_rows_fwd / bwd.
    dropout > 0 runs og_temporal_attn_long_dropout_fwd / bwd with a seed from _dropout_seed.
    causal=False (TemporalAttention's default, SDPA is_causal=False) runs og_temporal_attn_bidir_fwd / bwd at every T,
    with a seed only when dropout > 0; the per-pixel kernels and _time_attn_tiled are causal only."""

    @staticmethod
    def forward(ctx, x, freq, gamma, beta, k_cond, v_cond, n_head: int, scale: float, eps: float, dropout: float,
                causal: bool = True):
        _require_cuda(x, 'attention input')
        x = _rows_bf16(x)
        B, T, H, W, C = x.shape
        P = H * W
        s = _stream()
        q = torch.empty_like(x)
        _ln_rows_fwd(x, freq, gamma, beta, eps, q, B * T * P, C, P, T, s)
        y = torch.empty_like(x)
        bcast = k_cond is not None
        if bcast:
            kc = k_cond.detach().to(bf16).contiguous()
            vc = v_cond.detach().to(bf16).contiguous()
        else:
            kc = vc = q
        o = lse = seed = None
        if causal and not _time_attn_tiled(T, C, n_head, dropout):
            _lib.call('og_temporal_attn_fwd', q.data_ptr(), kc.data_ptr(), vc.data_ptr(), x.data_ptr(), y.data_ptr(),
                      B, T, P, C, n_head, scale, int(bcast), s)
        else:
            # the tiled kernels, which keep the attention output and log-sum-exp for the backward pass
            o = torch.empty_like(x)
            lse = torch.empty((B, n_head, P, T), dtype=f32, device=x.device)
            seed = _dropout_seed(x.device) if dropout > 0 else None
            if not causal:
                _lib.call('og_temporal_attn_bidir_fwd', q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o.data_ptr(),
                          x.data_ptr(), y.data_ptr(), lse.data_ptr(), B, T, P, C, n_head, scale, int(bcast), dropout,
                          _ptr(seed), s)
            elif dropout > 0:
                _lib.call('og_temporal_attn_long_dropout_fwd', q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o.data_ptr(),
                          x.data_ptr(), y.data_ptr(), lse.data_ptr(), B, T, P, C, n_head, scale, int(bcast), dropout,
                          seed.data_ptr(), s)
            else:
                _lib.call('og_temporal_attn_long_fwd', q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o.data_ptr(),
                          x.data_ptr(), y.data_ptr(), lse.data_ptr(), B, T, P, C, n_head, scale, int(bcast), s)
        ctx.cfg = (n_head, scale, eps, bcast, dropout, causal)
        ctx.save_for_backward(x, q, kc if bcast else None, vc if bcast else None, freq, gamma, o, lse, seed)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, q, kc, vc, freq, gamma, o, lse, seed = ctx.saved_tensors
        n_head, scale, eps, bcast, dropout, causal = ctx.cfg
        # the tiled backward, with the forward's dropout seed when it dropped
        if not causal:
            long_bwd, drop_args = 'og_temporal_attn_bidir_bwd', (dropout, _ptr(seed))
        elif dropout > 0:
            long_bwd, drop_args = 'og_temporal_attn_long_dropout_bwd', (dropout, seed.data_ptr())
        else:
            long_bwd, drop_args = 'og_temporal_attn_long_bwd', ()
        B, T, H, W, C = x.shape
        P = H * W
        s = _stream()
        dy = _rows_bf16(dy)
        dq = torch.empty_like(x)
        dkc = dvc = None
        delta = None if lse is None else torch.empty_like(lse)
        if bcast:
            dkc = _zeros((B, T, C), f32, x.device)
            dvc = _zeros((B, T, C), f32, x.device)
            if lse is None:
                _lib.call('og_temporal_attn_bwd', q.data_ptr(), kc.data_ptr(), vc.data_ptr(), dy.data_ptr(),
                          dq.data_ptr(), None, None, dkc.data_ptr(), dvc.data_ptr(), B, T, P, C, n_head, scale, 1, s)
            else:
                _lib.call(long_bwd, q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o.data_ptr(),
                          dy.data_ptr(), lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), None, None,
                          dkc.data_ptr(), dvc.data_ptr(), B, T, P, C, n_head, scale, 1, *drop_args, s)
            g1 = g2 = None
        else:
            dk, dv = torch.empty_like(x), torch.empty_like(x)
            if lse is None:
                _lib.call('og_temporal_attn_bwd', q.data_ptr(), q.data_ptr(), q.data_ptr(), dy.data_ptr(),
                          dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), None, None, B, T, P, C, n_head, scale, 0, s)
            else:
                _lib.call(long_bwd, q.data_ptr(), q.data_ptr(), q.data_ptr(), o.data_ptr(),
                          dy.data_ptr(), lse.data_ptr(), delta.data_ptr(), dq.data_ptr(),
                          dk.data_ptr(), dv.data_ptr(), None, None, B, T, P, C, n_head, scale, 0, *drop_args, s)
            g1, g2 = dk, dv
        dx = torch.empty_like(x)
        dgamma = _zeros(C, f32, x.device)
        dbeta = _zeros(C, f32, x.device)
        _ln_rows_bwd(x, freq, gamma, eps, dq, g1, g2, dy, dx, dgamma, dbeta, B * T * P, C, P, T, s)
        return dx, None, dgamma, dbeta, dkc, dvc, None, None, None, None, None


class _FfnFn(torch.autograd.Function):
    """out = FFN(x) + skip(x) — the ST block's ForwardBlock and its skip (attention.py:429-454, 472; misc.py:71-104):
        h = GroupNorm_G(x);  h = GELU(conv_i(h)) for every hidden layer;  y = conv_last(h)
    skip(x) = x (added inside the last conv's epilogue, its gradient inside the GN backward pass) or, when the block
    changes the width, the 1x1x1 ffn_skip conv as the second K segment of the last conv (x1 of og_conv3d_fwd).
    Inputs after `skip_b`: (weight, bias or None, packed operand) per conv, in order; `geoms` holds their ConvGeoms."""

    @staticmethod
    def forward(ctx, x, gn_w, gn_b, geoms, G: int, eps: float, skip_w, skip_b, *convs):
        _require_cuda(x, 'ffn input')
        x = _rows_bf16(x)
        B, T, H, W, C = x.shape
        V = T * H * W
        s = _stream()
        dev = x.device
        sums = _zeros((B, G, 2), torch.float64, dev, any(ctx.needs_input_grad))
        _lib.call('og_gn_stats', x.data_ptr(), B, V, C, G, sums.data_ptr(), s)
        A = torch.empty((B, C), dtype=f32, device=dev)
        Bc = torch.empty((B, C), dtype=f32, device=dev)
        mr = torch.empty((B, G, 2), dtype=f32, device=dev)
        hn = torch.empty_like(x)
        _lib.call('og_gn_act_fwd', x.data_ptr(), sums.data_ptr(), gn_w.data_ptr(), gn_b.data_ptr(), None, None, eps, G, 0,
                  hn.data_ptr(), A.data_ptr(), Bc.data_ptr(), mr.data_ptr(), B, V, C, s)
        ws = _workspace(dev, B * V * max(C, *(g.cout for g in geoms)) * 4)
        h, pre = hn, []                   # pre: the bf16 pre-activations u of the hidden layers (GELU backward)
        for i, geom in enumerate(geoms[:-1]):
            _, bias, packed = convs[3 * i:3 * i + 3]
            u = torch.empty((B, T, H, W, geom.cout), dtype=bf16, device=dev)
            _conv_call('fwd', 2.0 * B * V * geom.cout * geom.k_main, 'og_conv3d_fwd', h.data_ptr(), geom.cin, geom.kt,
                       geom.kh, geom.kw, geom.pt, geom.ph, geom.pw, None, 0, packed.data_ptr(), packed.shape[1],
                       _ptr(bias), None, None, u.data_ptr(), 0, B, T, H, W, geom.cout, ws.data_ptr(), ws.numel(), None, s)
            h = torch.empty_like(u)
            _lib.call('og_gelu_fwd', u.data_ptr(), h.data_ptr(), B * V, geom.cout, s)
            pre.append(u)
            pre.append(h)
        geom = geoms[-1]
        _, bias, packed = convs[-3:]
        y = torch.empty((B, T, H, W, geom.cout), dtype=bf16, device=dev)
        c1 = C if skip_w is not None else 0
        _conv_call('fwd', 2.0 * B * V * geom.cout * (geom.k_main + c1), 'og_conv3d_fwd', h.data_ptr(), geom.cin, geom.kt,
                   geom.kh, geom.kw, geom.pt, geom.ph, geom.pw, x.data_ptr() if c1 else None, c1, packed.data_ptr(),
                   packed.shape[1], _ptr(bias), _ptr(skip_b), None if c1 else x.data_ptr(), y.data_ptr(), 0, B, T, H, W,
                   geom.cout, ws.data_ptr(), ws.numel(), None, s)
        ctx.cfg = (geoms, G, tuple(convs[3 * i + 1] is not None for i in range(len(geoms))), skip_w is not None)
        ctx.save_for_backward(x, hn, A, Bc, mr, gn_w, gn_b, *convs[2::3], *pre)
        return y

    @staticmethod
    def backward(ctx, dy):
        geoms, G, has_bias, has_skip = ctx.cfg
        n = len(geoms)
        x, hn, A, Bc, mr, gn_w, gn_b, *rest = ctx.saved_tensors
        packs, pre = rest[:n], rest[n:]
        B, T, H, W, C = x.shape
        V = T * H * W
        s = _stream()
        dev = x.device
        dy = _rows_bf16(dy)
        ws = _workspace(dev, B * V * max(C, *(g.cout for g in geoms)) * 4)
        dh = torch.empty_like(x)
        S = _zeros((B, C, 2), f32, dev)
        grads = [None] * (3 * n)
        # per conv, last to first: data gradient -> GELU backward of the layer below it (or, below the first conv, the
        # GroupNorm backward reduction) -> weight (+ bias) gradient
        d_out = dy
        for i in reversed(range(n)):
            geom, packed = geoms[i], packs[i]
            cin, cout = geom.cin, geom.cout
            d_in = dh if i == 0 else torch.empty((B, T, H, W, cin), dtype=bf16, device=dev)
            _conv_call('dgrad', 2.0 * B * V * cout * geom.k_main, 'og_conv3d_dgrad', d_out.data_ptr(), cout, cout,
                       packed.data_ptr(), packed.shape[1], 0, geom.kt, geom.kh, geom.kw, geom.pt, geom.ph, geom.pw,
                       d_in.data_ptr(), 0, B, T, H, W, cin, ws.data_ptr(), ws.numel(), s)
            if i == 0:
                _lib.call('og_affine_act_bwd_reduce', dh.data_ptr(), x.data_ptr(), A.data_ptr(), Bc.data_ptr(), 0,
                          S.data_ptr(), B, V, C, *_scratch(dh), s)
                inp = hn
            else:
                u, inp = pre[2 * i - 2], pre[2 * i - 1]
                d_u = torch.empty_like(u)
                _lib.call('og_gelu_bwd', d_in.data_ptr(), u.data_ptr(), d_u.data_ptr(), B * V, cin, s)
            g = _zeros((cout, geom.ntaps * cin), f32, dev)
            fl = 2.0 * B * V * cout * geom.k_main
            if has_bias[i]:
                db = _zeros(cout, f32, dev)
                _conv_call('wgrad', fl, 'og_conv3d_wgrad_bias', d_out.data_ptr(), cout, inp.data_ptr(), cin, g.data_ptr(),
                           g.shape[1], geom.kt, geom.kh, geom.kw, geom.pt, geom.ph, geom.pw, B, T, H, W, db.data_ptr(),
                           cout, *_scratch(d_out), s)
                grads[3 * i + 1] = db
            else:
                _conv_call('wgrad', fl, 'og_conv3d_wgrad', d_out.data_ptr(), cout, inp.data_ptr(), cin, g.data_ptr(),
                           g.shape[1], geom.kt, geom.kh, geom.kw, geom.pt, geom.ph, geom.pw, B, T, H, W,
                           *_scratch(d_out), s)
            grads[3 * i] = g.view(cout, geom.kt, geom.kh, geom.kw, cin).permute(0, 4, 1, 2, 3)
            if i > 0:
                d_out = d_u
        add = dy
        dskip_w = dskip_b = None
        if has_skip:
            # the 1x1x1 shortcut: its data gradient is the `add` of the GN backward pass; its weight gradient reads x;
            # its bias gradient is the column sum of dy, as is that of the last conv's bias
            geom, packed = geoms[-1], packs[-1]
            cout = geom.cout
            add = torch.empty_like(x)
            _conv_call('dgrad', 2.0 * B * V * cout * C, 'og_conv3d_dgrad', dy.data_ptr(), cout, cout, packed.data_ptr(),
                       packed.shape[1], geom.kpad, 1, 1, 1, 0, 0, 0, add.data_ptr(), 0, B, T, H, W, C, ws.data_ptr(),
                       ws.numel(), s)
            g = _zeros((cout, C), f32, dev)
            if has_bias[-1]:
                dskip_b = grads[-2].clone()
                _conv_call('wgrad', 2.0 * B * V * cout * C, 'og_conv3d_wgrad', dy.data_ptr(), cout, x.data_ptr(), C,
                           g.data_ptr(), C, 1, 1, 1, 0, 0, 0, B, T, H, W, *_scratch(dy), s)
            else:
                dskip_b = _zeros(cout, f32, dev)
                _conv_call('wgrad', 2.0 * B * V * cout * C, 'og_conv3d_wgrad_bias', dy.data_ptr(), cout, x.data_ptr(), C,
                           g.data_ptr(), C, 1, 1, 1, 0, 0, 0, B, T, H, W, dskip_b.data_ptr(), cout, *_scratch(dy), s)
            dskip_w = g.view(cout, 1, 1, 1, C).permute(0, 4, 1, 2, 3)
        dgw = _zeros(C, f32, dev)
        dgb = _zeros(C, f32, dev)
        dx = torch.empty_like(x)
        _lib.call('og_gn_act_bwd', dh.data_ptr(), x.data_ptr(), A.data_ptr(), Bc.data_ptr(), S.data_ptr(), mr.data_ptr(),
                  gn_w.data_ptr(), gn_b.data_ptr(), None, G, 0, add.data_ptr(), dx.data_ptr(), dgw.data_ptr(),
                  dgb.data_ptr(), None, None, None, B, V, C, *_scratch(dy), s)
        return (dx, dgw, dgb, None, None, None, dskip_w, dskip_b, *grads)


def space_attention_res(x, freq, gamma, beta, n_head, scale, eps=1e-5, dropout=0.0, causal=False):
    return _SpaceAttnFn.apply(x, freq, gamma, beta, n_head, float(scale), float(eps), float(dropout), bool(causal))


def time_attention_res(x, freq, gamma, beta, n_head, scale, k_cond=None, v_cond=None, eps=1e-5, dropout=0.0,
                       causal=True):
    return _TimeAttnFn.apply(x, freq, gamma, beta, k_cond, v_cond, n_head, float(scale), float(eps), float(dropout),
                             bool(causal))


def ffn_res(x, gn_w, gn_b, convs, num_groups, eps=1e-5, skip_w=None, skip_b=None):
    """convs: (weight, bias or None, packed operand, ConvGeom) per conv of the FFN, first to last, a GELU after every
    conv but the last. skip_w / skip_b: the 1x1x1 ffn_skip conv, already fused into the last conv's packed operand
    (Conv3dParams.fuse_shortcut); without it the skip is x itself."""
    geoms = tuple(c[3] for c in convs)
    return _FfnFn.apply(x, gn_w, gn_b, geoms, num_groups, float(eps), skip_w, skip_b,
                        *(t for w, b, p, _ in convs for t in (w, b, p)))


# ------------------------------------------------------------------------------------------------
# row-wise linear layers on the conv GEMM kernel, embeddings, masked cross entropy
# ------------------------------------------------------------------------------------------------
def linear_rows(x2d: Tensor, weight: Tensor, bias: Optional[Tensor], packed: Tensor, out_f32: bool = False) -> Tensor:
    """y[rows][N] = x[rows][K] @ weight[N][K]^T + bias  (nn.Linear) as a 1x1x1 conv over `rows` voxels.
    weight: fp32 [N][K] (autograd leaf or view); packed: its bf16 copy [N][K]; K % 64 == 0."""
    rows, K = x2d.shape
    N = weight.shape[0]
    geom = ConvGeom(K, N, (1, 1, 1))
    x5 = x2d.reshape(1, 1, 1, rows, K).permute(0, 4, 1, 2, 3)
    y5 = _Conv3dFn.apply(x5, weight.view(N, K, 1, 1, 1), bias, None, None, None, packed, geom, out_f32, None)
    return y5.permute(0, 2, 3, 4, 1).reshape(rows, N)


class _EmbedAddFn(torch.autograd.Function):
    """tok_emb(tokens) + act_emb(act_id) broadcast over (h, w) -> (B,T,H,W,C) bf16 (dynamics.py:34-38, 55)."""

    @staticmethod
    def forward(ctx, tokens, act_id, tok_w, act_w):
        _require_cuda(tok_w, 'embedding weight')
        if tokens.dim() != 4:
            raise ValueError(f'embed_add: tokens must be (B, T, H, W), got {tuple(tokens.shape)}')
        if tuple(act_id.shape) != tuple(tokens.shape[:2]):
            # the reference adds act_emb (b,t,1,1,d) to tok_emb (b,t,h,w,d) (dynamics.py:55): mismatched t raises there
            raise ValueError(f'embed_add: act_id shape {tuple(act_id.shape)} does not match the (B, T) = '
                             f'{tuple(tokens.shape[:2])} of the tokens (one action per token frame)')
        B, T, H, W = tokens.shape
        C = tok_w.shape[1]
        tok = tokens.detach().to(torch.int64).contiguous()
        act = act_id.detach().to(torch.int64).contiguous()
        out = torch.empty((B, T, H, W, C), dtype=bf16, device=tok_w.device)
        _lib.call('og_embed_add_fwd', tok.data_ptr(), act.data_ptr(), tok_w.data_ptr(), act_w.data_ptr(), out.data_ptr(),
                  B * T * H * W, H * W, C, tok_w.shape[0], act_w.shape[0], _stream())
        ctx.save_for_backward(tok, act)
        ctx.shapes = (tok_w.shape, act_w.shape, H * W)
        return out

    @staticmethod
    def backward(ctx, dy):
        tok, act = ctx.saved_tensors
        ts, as_, hw = ctx.shapes
        dy = _rows_bf16(dy)
        dtw = _zeros(ts, f32, dy.device)
        daw = _zeros(as_, f32, dy.device)
        _lib.call('og_embed_add_bwd', tok.data_ptr(), act.data_ptr(), dy.data_ptr(), dtw.data_ptr(), daw.data_ptr(),
                  tok.numel(), hw, ts[1], ts[0], as_[0], _stream())
        return None, None, dtw, daw


def embed_add(tokens, act_id, tok_w, act_w):
    return _EmbedAddFn.apply(tokens, act_id, tok_w, act_w)


class _MaskedCeFn(torch.autograd.Function):
    """cross_entropy(logits[mask], target[mask]) with mean reduction (dynamics.py:89-97)."""

    @staticmethod
    def forward(ctx, logits2d, target, mask):
        rows, V = logits2d.shape
        lg = logits2d if (logits2d.dtype == bf16 and logits2d.is_contiguous()) else logits2d.to(bf16).contiguous()
        tgt = target.detach().reshape(-1).to(torch.int64).contiguous()
        msk = mask.detach().reshape(-1).to(torch.uint8).contiguous()
        row_lse = torch.empty(rows, dtype=f32, device=lg.device)
        stats = torch.zeros(2, dtype=f32, device=lg.device)
        _lib.call('og_masked_ce_fwd', lg.data_ptr(), tgt.data_ptr(), msk.data_ptr(), rows, V, row_lse.data_ptr(),
                  stats.data_ptr(), _stream())
        ctx.save_for_backward(lg, tgt, msk, row_lse, stats)
        return stats[0] / stats[1]

    @staticmethod
    def backward(ctx, g):
        lg, tgt, msk, row_lse, stats = ctx.saved_tensors
        gs = g.detach().to(f32).contiguous()
        dl = torch.empty_like(lg)
        _lib.call('og_masked_ce_bwd', lg.data_ptr(), tgt.data_ptr(), msk.data_ptr(), row_lse.data_ptr(), stats.data_ptr(),
                  gs.data_ptr(), dl.data_ptr(), lg.shape[0], lg.shape[1], _stream())
        return dl, None, None


def masked_cross_entropy(logits2d, target, mask):
    return _MaskedCeFn.apply(logits2d, target, mask)


def maskgit_sample(logits_last: Tensor, uniforms: Tensor, schedule: Tensor, temp: float = 1.0, masked_tok: int = 0
                   ) -> Tensor:
    """All MaskGIT sampling iterations of DynamicsModel.generate (genie/dynamics.py:136-163) on the last frame's logits
    (b, h, w, V): softmax -> CDF once (og_softmax_cdf), then one launch that runs every iteration (og_maskgit_sample).
    uniforms: (steps, b*h*w) in [0, 1); schedule: (steps,) tokens to fix per iteration. Returns code (b, h, w) int64."""
    _require_cuda(logits_last, 'logits')
    b, h, w, V = logits_last.shape
    P = h * w
    lg = logits_last.detach()
    if lg.dtype not in (bf16, f32) or not lg.is_contiguous():
        lg = lg.float().contiguous()
    dev = lg.device
    s = _stream()
    cdf = torch.empty((b * P, V), dtype=f32, device=dev)
    row_stats = torch.empty((b * P, 2), dtype=f32, device=dev)
    lg_f32, inv_temp = int(lg.dtype == f32), 1.0 / float(temp)
    _lib.call('og_softmax_cdf', lg.data_ptr(), lg_f32, b * P, V, inv_temp, cdf.data_ptr(), row_stats.data_ptr(), s)
    steps = int(schedule.numel())
    u = uniforms.detach().to(device=dev, dtype=f32).reshape(steps, b * P).contiguous()
    sch = schedule.detach().to(device=dev, dtype=torch.int32).contiguous()
    code = torch.full((b, P), int(masked_tok), dtype=torch.int64, device=dev)
    mask = torch.ones((b, P), dtype=torch.uint8, device=dev)
    _lib.call('og_maskgit_sample', cdf.data_ptr(), lg.data_ptr(), lg_f32, inv_temp, row_stats.data_ptr(), u.data_ptr(),
              sch.data_ptr(), steps, b, P, V, code.data_ptr(), mask.data_ptr(), s)
    return code.view(b, h, w), mask.view(b, h, w)


# ------------------------------------------------------------------------------------------------
# fused VideoResidualBlock (no down-sampling): GN+SiLU -> conv -> GN+SiLU -> conv (+) 1x1x1 shortcut (+) add
# ------------------------------------------------------------------------------------------------
class _ResBlockFn(torch.autograd.Function):
    """One autograd node for the whole block (genie/module/video.py:539-656) so that
      * GroupNorm statistics of each conv output come out of the producing GEMM's epilogue (gn_sums),
      * the shortcut's data gradient is added inside the last backward apply pass (no stand-alone add),
    leaving per block: 2 apply passes forward, 2 apply passes backward, 2 column-sum passes, and the GEMMs."""

    @staticmethod
    def forward(ctx, x, x_sums, g1w, g1b, w1, b1, g2w, g2b, w2, b2, wres, bres, packed1, packed2, geom1: ConvGeom,
                geom2: ConvGeom, G: int, eps: float, act: int = 1):
        _require_cuda(x, 'residual block input')
        xi = to_internal(x, bf16)
        B, C0, T, H, W = xi.shape
        C1 = geom1.cout
        V = T * H * W
        s = _stream()
        dev = xi.device
        rec = any(ctx.needs_input_grad)
        if x_sums is None:
            x_sums = _zeros((B, G, 2), torch.float64, dev, rec)
            _lib.call('og_gn_stats', xi.data_ptr(), B, V, C0, G, x_sums.data_ptr(), s)
        mr = torch.empty((2, B, G, 2), dtype=f32, device=dev)
        A1, B1 = torch.empty((B, C0), dtype=f32, device=dev), torch.empty((B, C0), dtype=f32, device=dev)
        A2, B2 = torch.empty((B, C1), dtype=f32, device=dev), torch.empty((B, C1), dtype=f32, device=dev)
        a1 = empty_internal(B, C0, T, H, W, bf16, dev)
        _lib.call('og_gn_act_fwd', xi.data_ptr(), x_sums.data_ptr(), g1w.data_ptr(), g1b.data_ptr(), None, None, eps, G, act,
                  a1.data_ptr(), A1.data_ptr(), B1.data_ptr(), mr[0].data_ptr(), B, V, C0, s)
        ws = _workspace(dev, B * V * C1 * 4)
        fuse_stats = G == 1
        sums2 = _zeros((B, G, 2), torch.float64, dev, rec)
        h1 = empty_internal(B, C1, T, H, W, bf16, dev)
        _conv_call('fwd', 2.0 * B * V * C1 * geom1.k_main, 'og_conv3d_fwd', a1.data_ptr(), C0, geom1.kt, geom1.kh,
                   geom1.kw, geom1.pt, geom1.ph, geom1.pw, None, 0, packed1.data_ptr(), packed1.shape[1], _ptr(b1), None,
                   None, h1.data_ptr(), 0, B, T, H, W, C1, ws.data_ptr(), ws.numel(),
                   sums2.data_ptr() if fuse_stats else None, s)
        if not fuse_stats:
            _lib.call('og_gn_stats', h1.data_ptr(), B, V, C1, G, sums2.data_ptr(), s)
        a2 = empty_internal(B, C1, T, H, W, bf16, dev)
        _lib.call('og_gn_act_fwd', h1.data_ptr(), sums2.data_ptr(), g2w.data_ptr(), g2b.data_ptr(), None, None, eps, G, act,
                  a2.data_ptr(), A2.data_ptr(), B2.data_ptr(), mr[1].data_ptr(), B, V, C1, s)
        y = empty_internal(B, C1, T, H, W, bf16, dev)
        y_sums = _zeros((B, 1, 2), torch.float64, dev, rec)
        _conv_call('fwd', 2.0 * B * V * C1 * (geom2.k_main + C0), 'og_conv3d_fwd', a2.data_ptr(), C1, geom2.kt, geom2.kh,
                   geom2.kw, geom2.pt, geom2.ph, geom2.pw, xi.data_ptr(), C0, packed2.data_ptr(), packed2.shape[1],
                   _ptr(b2), _ptr(bres), None, y.data_ptr(), 0, B, T, H, W, C1, ws.data_ptr(), ws.numel(),
                   y_sums.data_ptr(), s)
        ctx.cfg = (geom1, geom2, G, b1 is not None, b2 is not None, bres is not None, act)
        ctx.save_for_backward(xi, a1, h1, a2, A1, B1, A2, B2, mr, g1w, g1b, g2w, g2b, packed1, packed2)
        ctx.mark_non_differentiable(y_sums)
        ctx.set_materialize_grads(False)     # else autograd fills a zero "gradient" for y_sums in every backward (40 launches)
        return y, y_sums

    @staticmethod
    def backward(ctx, dy, _dsums):
        xi, a1, h1, a2, A1, B1, A2, B2, mr, g1w, g1b, g2w, g2b, packed1, packed2 = ctx.saved_tensors
        geom1, geom2, G, has_b1, has_b2, has_bres, act = ctx.cfg
        B, C0, T, H, W = xi.shape
        C1 = geom1.cout
        V = T * H * W
        s = _stream()
        dev = xi.device
        dyb = _as_bf16_rows(dy, C1, C1)
        ws = _workspace(dev, B * V * max(C0, C1) * 4)
        ld2 = packed2.shape[1]

        def wgrad(dyt, cout, xin, cin, g, dbias=None):
            gr = _zeros((cout, g.ntaps * cin), f32, dev)
            if dbias is None:
                _conv_call('wgrad', 2.0 * B * V * cout * cin * g.ntaps, 'og_conv3d_wgrad', dyt.data_ptr(), cout,
                           xin.data_ptr(), cin, gr.data_ptr(), gr.shape[1], g.kt, g.kh, g.kw, g.pt, g.ph, g.pw, B, T, H, W,
                           *_scratch(dyt), s)
            else:       # + the bias gradient (column sums of dy) out of the same tensor-core pass
                _conv_call('wgrad', 2.0 * B * V * cout * cin * g.ntaps, 'og_conv3d_wgrad_bias', dyt.data_ptr(), cout,
                           xin.data_ptr(), cin, gr.data_ptr(), gr.shape[1], g.kt, g.kh, g.kw, g.pt, g.ph, g.pw, B, T, H, W,
                           dbias.data_ptr(), cout, *_scratch(dyt), s)
            return gr.view(cout, g.kt, g.kh, g.kw, cin).permute(0, 4, 1, 2, 3)

        gone = ConvGeom(C0, C1, (1, 1, 1))
        db2 = _zeros(C1, f32, dev)
        dw2 = wgrad(dyb, C1, a2, C1, geom2)
        dwres = wgrad(dyb, C1, xi, C0, gone, dbias=db2)   # 1 tap: spare accumulator columns
        # conv2 data gradient, then the GN2 backward
        S2 = _zeros((B, C1, 2), f32, dev)
        d_a2 = empty_internal(B, C1, T, H, W, bf16, dev)
        _conv_call('dgrad', 2.0 * B * V * C1 * geom2.k_main, 'og_conv3d_dgrad', dyb.data_ptr(), C1, C1, packed2.data_ptr(),
                   ld2, 0, geom2.kt, geom2.kh, geom2.kw, geom2.pt, geom2.ph, geom2.pw, d_a2.data_ptr(), 0, B, T, H, W, C1,
                   ws.data_ptr(), ws.numel(), s)
        small = _zeros((3, C1), f32, dev)              # dgamma2, dbeta2, db1 in one fill
        dg2w, dg2b, db1 = small[0], small[1], small[2]
        d_h1 = empty_internal(B, C1, T, H, W, bf16, dev)
        _gn_bwd(d_a2, h1, A2, B2, S2, mr[1], g2w, g2b, G, act, None, d_h1, dg2w, dg2b, db1 if has_b1 else None, B, V, C1, s)
        dw1 = wgrad(d_h1, C1, a1, C0, geom1)
        dx = None
        dg1w, dg1b = _zeros(C0, f32, dev), _zeros(C0, f32, dev)
        dx_res = empty_internal(B, C0, T, H, W, bf16, dev)
        # conv1 data gradient; GN1 backward reduction; shortcut data gradient; GN1 backward apply adds both
        S1 = _zeros((B, C0, 2), f32, dev)
        d_a1 = empty_internal(B, C0, T, H, W, bf16, dev)
        _conv_call('dgrad', 2.0 * B * V * C1 * geom1.k_main, 'og_conv3d_dgrad', d_h1.data_ptr(), C1, C1,
                   packed1.data_ptr(), packed1.shape[1], 0, geom1.kt, geom1.kh, geom1.kw, geom1.pt, geom1.ph, geom1.pw,
                   d_a1.data_ptr(), 0, B, T, H, W, C0, ws.data_ptr(), ws.numel(), s)
        _lib.call('og_affine_act_bwd_reduce', d_a1.data_ptr(), xi.data_ptr(), A1.data_ptr(), B1.data_ptr(), act,
                  S1.data_ptr(), B, V, C0, *_scratch(d_a1), s)
        _conv_call('dgrad', 2.0 * B * V * C1 * C0, 'og_conv3d_dgrad', dyb.data_ptr(), C1, C1, packed2.data_ptr(), ld2,
                   geom2.k_main, 1, 1, 1, 0, 0, 0, dx_res.data_ptr(), 0, B, T, H, W, C0, ws.data_ptr(), ws.numel(), s)
        # (the input gradient is always produced: its pass is also what emits dgamma1 / dbeta1)
        dx = empty_internal(B, C0, T, H, W, bf16, dev)
        _gn_bwd(d_a1, xi, A1, B1, S1, mr[0], g1w, g1b, G, act, dx_res, dx, dg1w, dg1b, None, B, V, C0, s, reduce=False)
        return (dx, None, dg1w, dg1b, dw1, db1 if has_b1 else None, dg2w, dg2b, dw2, db2 if has_b2 else None, dwres,
                (db2.clone() if has_b2 else db2) if has_bres else None, None, None, None, None, None, None, None)


def residual_block(x, x_sums, g1w, g1b, w1, b1, g2w, g2b, w2, b2, wres, bres, packed1, packed2, geom1, geom2, G, eps,
                   act='silu'):
    return _ResBlockFn.apply(x, x_sums, g1w, g1b, w1, b1, g2w, g2b, w2, b2, wres, bres, packed1, packed2, geom1, geom2, G,
                             float(eps), act_code(act))
