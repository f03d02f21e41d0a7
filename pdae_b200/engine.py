"""Static launch plans over the C-ABI kernels.

A ``Plan`` is recorded once per (module, input shape, precision): a flat list of native calls on
pre-assigned device buffers (liveness-based reuse of one arena), so a forward pass is a tight loop of
ctypes calls on the current CUDA stream -- no allocation, no host sync, legal under CUDA-graph capture.
PyTorch is used here only for device memory and streams.

Precision modes
  * ``fp32``: every contraction on CUDA cores in fp32 (pdae_conv2d_simt / pdae_attention_simt).  This is
    the mode that holds rtol 1e-3 / atol 1e-4 against the CPU oracle.
  * ``bf16``: convolutions and attention GEMMs whose shapes allow it run on the wgmma tensor-core kernels
    with bf16 operands and fp32 accumulation (pdae_conv_tc2_* / pdae_gemm_tc2_*, and pdae_conv_tc3_* with
    GroupNorm-apply / SiLU fused into the operand path); the residual stream is bf16, GroupNorm statistics,
    embeddings and the DDIM update stay fp32.
  * ``bf16x3``: the same tensor-core kernels on split operands (a = hi + lo, three bf16 products per term)
    for fp32-grade results; the residual stream and GroupNorm inputs stay fp32.

Deterministic plans (``Plan(..., deterministic=True)``; the modules record them while
``torch.are_deterministic_algorithms_enabled()``): every cross-CTA reduction -- GroupNorm statistics, split-K Linears -- runs
on kernels without float atomics whose partial results have fixed slots summed in a fixed order, so a replay gives the same
bits for the same inputs.  The default plans keep the atomic kernels.  A deterministic backward plan (train.py) does the same for
the weight / bias / GroupNorm / embedding gradients and the split-K data gradients; every gradient buffer is then written by
plain stores (Plan.new_grad), so it needs no zeroed accumulator.
"""
from __future__ import annotations

import ctypes
import os
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from . import _native
from ._native import PDAE_BF16, PDAE_F32, RESAMPLE_DOWN2, RESAMPLE_NONE, RESAMPLE_UP2

_DT = {torch.float32: PDAE_F32, torch.bfloat16: PDAE_BF16}
_STREAM = object()  # placeholder replaced by the current stream at run time
FUSE_DESC_LEN = 10  # int64 slots of an image head's fused-update descriptor (include/pdae_b200.h: pdae_conv_tc2_set_head_fuse)

_default_precision = "bf16"
# "fp32"   : CUDA-core fp32 arithmetic everywhere (parity / training mode)
# "bf16"   : wgmma bf16 MMAs, bf16 activations and residual stream (the fast mode; stated tolerance rel-L2 <= 2e-2)
# "bf16x3" : wgmma bf16 MMAs on split operands (a = hi + lo, three products per term), fp32 residual stream and GroupNorm
#            inputs: fp32-grade results (meets the fp32 tolerance) at ~3x the MMA work of "bf16"
PRECISIONS = ("fp32", "bf16", "bf16x3")


def set_default_precision(p: str) -> None:
    global _default_precision
    if p not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}")
    _default_precision = p


def get_default_precision() -> str:
    return _default_precision


class Buf:
    """A device buffer known to a plan: either plan-owned (arena) or fixed (parameter / caller tensor)."""
    __slots__ = ("shape", "dtype", "tensor", "first", "last", "fixed", "keep", "name", "_block", "split3", "tc_copy")

    def __init__(self, shape, dtype, tensor=None, name=""):
        self.shape = tuple(int(s) for s in shape)
        self.dtype = dtype
        self.tensor = tensor
        self.fixed = tensor is not None
        self.first = None
        self.last = None
        self.keep = False
        self.name = name
        self.split3 = False   # "bf16x3" activation: last dim holds three bf16 channel blocks [hi | lo | hi]
        self.tc_copy = None   # training forward: the bf16 tensor-core copy of this fp32 activation (Plan.conv, train_tc)

    @property
    def nbytes(self) -> int:
        n = torch.empty((), dtype=self.dtype).element_size()
        for s in self.shape:
            n *= s
        return n

    def at(self, elem_offset: int) -> "BufView":
        return BufView(self, elem_offset)


class BufView:
    __slots__ = ("buf", "off")

    def __init__(self, buf: Buf, off: int):
        self.buf, self.off = buf, int(off)

    def at(self, elem_offset: int) -> "BufView":
        return BufView(self.buf, self.off + elem_offset)


class Packed:
    """A derived (re-laid-out / converted) copy of parameters, refreshed when a source changes."""

    def __init__(self, sources: Sequence[torch.Tensor], fn: Callable[[], torch.Tensor]):
        self.sources = list(sources)
        self.fn = fn
        self.tensor = fn().contiguous()
        self.stamp = self._stamp()

    def _stamp(self):
        return tuple((s.data_ptr(), s._version) for s in self.sources)

    def refresh(self, force: bool = False) -> None:
        """Re-pack when a source's (storage, version) changed -- or unconditionally (`force`): writes through `p.data`
        (the reference trainers' EMA loop, train_representation_learning.py:192-212) and raw-pointer writes bump no
        version counter, so every sampling loop / graph capture forces one refresh (Plan.run_prologue)."""
        st = self._stamp()
        if force or st != self.stamp:
            with torch.inference_mode(False), torch.no_grad(), _fully_written():
                self.tensor.copy_(self.fn())
            self.stamp = st


class _fully_written:
    """Within: PyTorch does not fill new tensors first (torch.utils.deterministic.fill_uninitialized_memory, which the
    deterministic mode turns on).  A pack's temporaries are written in full by the ops that make them, and a training step
    re-packs every updated weight: the fill would add a kernel per temporary, several hundred per step."""

    def __enter__(self):
        self.was = torch.utils.deterministic.fill_uninitialized_memory
        torch.utils.deterministic.fill_uninitialized_memory = False

    def __exit__(self, *exc):
        torch.utils.deterministic.fill_uninitialized_memory = self.was


def split3_weights(w: torch.Tensor) -> torch.Tensor:
    """[Cout][Cin][taps] fp32 -> [taps][Cout][3*Cin] bf16 = [W_hi | W_hi | W_lo] (pairs with activations [a_hi | a_lo | a_hi])."""
    w = w.float()
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, hi, lo], dim=1).permute(2, 0, 1).contiguous()


class CoefSpec:
    """GroupNorm coefficients not yet computed: the per-channel statistics and affine / AdaGN operands a later gn_apply
    needs (Plan.gn_coef in fused-statistics mode)."""
    __slots__ = ("stats1", "C1", "stats2", "C2", "gamma", "beta", "B", "HW", "emb", "emb_ld", "embz", "embz_ld")

    def __init__(self, stats1, C1, stats2, C2, gamma, beta, B, HW, emb, emb_ld, embz, embz_ld):
        self.stats1, self.C1, self.stats2, self.C2, self.gamma, self.beta = stats1, C1, stats2, C2, gamma, beta
        self.B, self.HW, self.emb, self.emb_ld, self.embz, self.embz_ld = B, HW, emb, emb_ld, embz, embz_ld


class Plan:
    def __init__(self, device: torch.device, precision: Optional[str] = None, check_device: bool = True,
                 deterministic: bool = False):
        if check_device:  # False only in CPU unit tests of the recording / buffer-assignment logic (a plan cannot run there)
            _native.require_device()
        self.device = device
        self.precision = precision or _default_precision
        if self.precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}")
        self.x3 = self.precision == "bf16x3"                     # split-operand tensor-core mode (fp32-grade results)
        self.tc = self.precision in ("bf16", "bf16x3")
        # residual stream (block outputs / skip tensors) kept in bf16 instead of fp32: halves the HBM bytes of the
        # bandwidth-bound top-level layers.  "bf16" precision only.
        self.stream_bf16 = self.precision == "bf16"
        self.L = _native.lib()
        self.det = bool(deterministic)   # record the deterministic kernels (module docstring)
        self._det_handles: list = []     # (op index, set_deterministic, workspace query, handle): DET_OPS, switched at finalize
        self._det_ws = None
        self.ops: List[Tuple[str, list]] = []
        # ops recorded inside `with P.prologue():` depend only on inputs that are constant over a sampling loop (z):
        # a loop runs them once (run_prologue) and replays the remaining ops per step (run(prologue=False))
        self.op_pro: List[bool] = []
        self._in_prologue = False
        self.bufs: List[Buf] = []
        self.packed: List[Packed] = []
        self.params: List[Tuple[torch.Tensor, int]] = []
        self._pack_cache: Dict[tuple, Buf] = {}
        self._compiled = None
        self._tc2_handles: List[ctypes.c_void_p] = []
        self._tc3_handles: List[ctypes.c_void_p] = []
        self._wg_handles: List[ctypes.c_void_p] = []
        self._nplan_handles: List[ctypes.c_void_p] = []
        self._native_plans: dict = {}
        self.head_fuse: Dict[str, Buf] = {}   # image heads whose epilogue can run the DDIM update (set by a sampling loop)
        # training forward plans (fp32, every intermediate kept for the backward): the precision of the eligible convs on the
        # tensor cores.  None: CUDA cores; "bf16x3": split operands (a [hi | lo | hi] copy of the fp32 activation feeds conv_tc2);
        # "bf16": a plain bf16 copy feeds conv_tc2 (autocast training).  The fp32 activation the backward needs stays as it is.
        self.train_tc: Optional[str] = None
        self.n_launch = 0
        self.keep_all = False
        self.dropout_masks: list = []   # (block, mask buffer, p): filled by the trainer before every training forward
        self.last_sums = None
        self._stats_arena = Buf((1,), torch.float32, None, "stats_arena")  # sized at finalize
        self._stats_arena.keep = True
        self._stats_arena.first = 0
        self._stats_arena.last = 0
        self.bufs.append(self._stats_arena)
        self._stats_elems = 0
        self.graph = None
        self.flops: List[float] = []  # algorithmic FLOPs (2*MACs) per recorded op, 0 for non-contraction ops
        self._launches: Dict[int, int] = {}   # op index -> kernel launches, where the op's shape decides it (Plan.call)

    # ---- buffers ----------------------------------------------------------------------------
    def new(self, shape, dtype=torch.float32, name="") -> Buf:
        b = Buf(shape, dtype, None, name)
        if self.keep_all:  # training plans: every intermediate may be needed by the backward plan -> no recycling
            b.keep = True
        self.bufs.append(b)
        return b

    def new_zeroed(self, nelems: int) -> "BufView":
        """fp32 scratch of `nelems` elements inside the arena that ONE memset per replay zeroes (gradient / statistics
        accumulators written with atomics)."""
        off = self._stats_elems
        self._stats_elems += int(nelems)
        return BufView(self._stats_arena, off)

    def new_grad(self, nelems: int) -> "BufView":
        """fp32 gradient buffer of `nelems` elements: in the zeroed arena (new_zeroed) for the atomic kernels of a default plan;
        private storage, written by plain stores and read after the run, in a deterministic plan."""
        if not self.det:
            return self.new_zeroed(nelems)
        b = self.new((int(nelems),), torch.float32, "grad")
        b.keep = True
        return BufView(b, 0)

    def det_workspace(self, nbytes: int, what: str) -> Buf:
        """Arena scratch for the slots of a deterministic op (`nbytes` from its *_workspace_bytes query)."""
        _native.check(min(int(nbytes), 0), what)
        return self.new((max(int(nbytes), 16) // 4,), torch.float32, "det_slots")

    def fixed(self, t: torch.Tensor) -> Buf:
        assert t.is_contiguous(), "plan tensors must be contiguous"
        return Buf(t.shape, t.dtype, t)

    def param(self, p: Optional[torch.Tensor]) -> Optional[Buf]:
        """A parameter consumed in place (fp32, contiguous); tracked so a moved parameter invalidates the plan."""
        if p is None:
            return None
        if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
            raise _native.NativeError("pdae_b200 modules need contiguous fp32 CUDA parameters (no CPU fallback)")
        self.params.append((p, p.data_ptr()))
        return Buf(p.shape, p.dtype, p.detach())

    def pack(self, key: tuple, sources: Sequence[torch.Tensor], fn: Callable[[], torch.Tensor]) -> Buf:
        if key in self._pack_cache:
            return self._pack_cache[key]
        for s in sources:
            if not s.is_cuda:
                raise _native.NativeError("pdae_b200 modules need CUDA parameters (no CPU fallback)")
        with torch.inference_mode(False), torch.no_grad():  # never create inference tensors: plans outlive the caller's mode
            pk = Packed([s for s in sources], fn)
        self.packed.append(pk)
        b = Buf(pk.tensor.shape, pk.tensor.dtype, pk.tensor)
        self._pack_cache[key] = b
        return b

    # ---- recording --------------------------------------------------------------------------
    def prologue(self):
        """Context manager: ops recorded inside are step-invariant (SURVEY.md §8(f) row 2).  Every buffer they produce
        for the per-step ops must be `keep` (private storage) -- asserted at finalize."""
        plan = self

        class _Ctx:
            def __enter__(self):
                plan._in_prologue = True

            def __exit__(self, *exc):
                plan._in_prologue = False
        return _Ctx()

    def call(self, fn: str, *args, flops: float = 0.0, launches: Optional[int] = None) -> None:
        """Record one native call.  launches: the kernels it runs when that depends on its shape (otherwise _LAUNCHES / 1)."""
        idx = len(self.ops)
        if launches is not None:
            self._launches[idx] = int(launches)
        self.flops.append(float(flops))
        self.op_pro.append(self._in_prologue)
        flat = []
        for a in args:
            flat.extend(a if isinstance(a, tuple) else (a,))
        for a in flat:
            b = a.buf if isinstance(a, BufView) else a
            if isinstance(b, Buf) and not b.fixed:
                if b.first is None:
                    b.first = idx
                b.last = idx
        self.ops.append((fn, list(args)))

    # ---- finalisation -----------------------------------------------------------------------
    def finalize(self) -> "Plan":
        with torch.inference_mode(False):
            return self._finalize()

    def _finalize(self) -> "Plan":
        self._stats_arena.shape = (max(self._stats_elems, 4),)
        if self._stats_elems:
            self.ops.insert(0, ("zero", [self._stats_arena, ctypes.c_int64(self._stats_elems * 4), _STREAM]))
            self.flops.insert(0, 0.0)
            self.op_pro.insert(0, False)
            self._launches = {i + 1: n for i, n in self._launches.items()}
            for b in self.bufs:  # op indices shift by one
                if b is not self._stats_arena and b.first is not None:
                    b.first += 1
                    b.last += 1
            self._stats_arena.last = len(self.ops) - 1
        starts: Dict[int, List[Buf]] = {}
        ends: Dict[int, List[Buf]] = {}
        for b in self.bufs:
            if b.first is None:
                continue
            starts.setdefault(b.first, []).append(b)
            if not b.keep:
                ends.setdefault(b.last, []).append(b)
        free: List[torch.Tensor] = []
        self.arena_bytes = 0
        # `keep` buffers are the plan's inputs/outputs: the caller writes/reads them OUTSIDE the op sequence, so their
        # live range is the whole plan -- they get private storage and never touch the recycling pool.
        for b in self.bufs:
            if b.keep and b.first is not None:
                b.tensor = torch.empty(max(b.nbytes, 16), dtype=torch.uint8, device=self.device)[: b.nbytes].view(
                    b.dtype).view(b.shape)
                self.arena_bytes += b.nbytes
        for i in range(len(self.ops)):
            for b in starts.get(i, []):
                if b.keep:
                    continue
                need = max(b.nbytes, 16)
                best = None
                for j, blk in enumerate(free):
                    if blk.numel() >= need and (best is None or blk.numel() < free[best].numel()):
                        best = j
                if best is not None and free[best].numel() <= 2 * need + 4096:
                    blk = free.pop(best)
                else:
                    blk = torch.empty(need, dtype=torch.uint8, device=self.device)
                    self.arena_bytes += need
                b.tensor = blk[: b.nbytes].view(b.dtype).view(b.shape)
                b._block = blk  # type: ignore[attr-defined]
            for b in ends.get(i, []):
                free.append(b._block)  # type: ignore[attr-defined]
        if self.det:
            bad = sorted({fn for fn, _ in self.ops} & NONDET_OPS)
            if bad:
                raise ValueError(f"a deterministic plan cannot record {bad}: their kernels reduce with float atomics")
        compiled = []
        for fn, args in self.ops:
            if self.det and fn in DET_OPS:   # the handle each of these ops compiles to is switched to its DET kernels below
                setter, query = det_entry_points(fn)
                self._det_handles.append((len(compiled), getattr(self.L, setter), getattr(self.L, query)))
            if fn == "conv_tc2":
                compiled.append(self._compile_tc2(args))
                continue
            if fn == "gemm_tc2":
                compiled.append(self._compile_gemm(args))
                continue
            if fn == "gemm_tc2_softmax":
                compiled.append(self._compile_gemm_softmax(args))
                continue
            if fn == "gemm_tc2_major":
                compiled.append(self._compile_gemm_major(args))
                continue
            if fn == "gemm_tc2_softmax_grad":
                compiled.append(self._compile_gemm_softmax_grad(args))
                continue
            if fn == "conv_tc2_skip":
                compiled.append(self._compile_tc2_skip(args))
                continue
            if fn == "conv_tc3":
                compiled.append(self._compile_tc3(args))
                continue
            if fn in ("wgrad_tc", "wgrad_tc_bf16"):
                compiled.append(self._compile_wgrad(args, split=fn == "wgrad_tc"))
                continue
            if fn in ("conv_tc2_s2", "conv_tc2_s2_dgrad", "wgrad_tc_bf16_s2"):
                compiled.append(self._compile_s2(fn, args))
                continue
            if fn == "conv_tc2_splitk":
                compiled.append(self._compile_splitk(args))
                continue
            cargs = []
            sidx = -1
            for k, a in enumerate(args):
                if a is _STREAM:
                    sidx = k
                    cargs.append(None)
                else:
                    cargs.append(self._resolve(a))
            compiled.append((getattr(self.L, "pdae_" + fn), cargs, sidx, fn))
        extra = {}   # op index -> launches a deterministic op adds (the reduction of its slots)
        if self._det_handles:
            # one workspace serves every tensor-core op of the plan: each op's slots live only inside its own run, and the ops run
            # one after another on one stream
            self._det_handles = [(i, st, q, compiled[i][1][0]) for i, st, q in self._det_handles]
            need = [int(q(h)) for _, _, q, h in self._det_handles]
            if min(need) < 0:
                _native.check(min(need), "det_workspace_bytes")
            self._det_ws = torch.empty(max(max(need), 16), dtype=torch.uint8, device=self.device)
            for (i, setter, _, h), n in zip(self._det_handles, need):
                _native.check(setter(h, ctypes.c_void_p(self._det_ws.data_ptr()), ctypes.c_int64(self._det_ws.numel())),
                              setter.__name__)
                extra[i] = 1 if (n > 0 or self.ops[i][0] == "conv_tc2_splitk") else 0
        self._compiled = compiled
        self._pro_idx = [i for i, p in enumerate(self.op_pro) if p]
        self._main_idx = [i for i, p in enumerate(self.op_pro) if not p]
        # PDAE_NATIVE_PLAN=1: replay through the C-ABI plan executor (pdae_plan_*): one foreign call per pass instead of one
        # ctypes call per op.  Off by default (the Python loop is the path the GPU suite of this round validated).
        self._native_plans = {}
        if os.environ.get("PDAE_NATIVE_PLAN", "0") == "1":
            self._native_plans = {"pro": self._build_native(self._pro_idx), "main": self._build_native(self._main_idx)}
        for b in self.bufs:  # a recycled buffer must not carry data from the prologue into the per-step ops
            if b.first is not None and not b.keep and not b.fixed and self.op_pro[b.first] and not self.op_pro[b.last]:
                raise AssertionError(f"plan buffer {b.name!r} crosses the prologue boundary but is not `keep`")
        self.n_launch = sum(self._launches.get(i, _LAUNCHES.get(fn, 1)) + extra.get(i, 0)
                            for i, ((fn, _), p) in enumerate(zip(self.ops, self.op_pro)) if not p)
        return self

    @staticmethod
    def _resolve(a):
        if isinstance(a, Buf):
            return ctypes.c_void_p(a.tensor.data_ptr())
        if isinstance(a, BufView):
            return ctypes.c_void_p(a.buf.tensor.data_ptr() + a.off * a.buf.tensor.element_size())
        return a

    def _compile_tc2(self, args):
        fuse = args[15] if len(args) > 15 else None
        x, w, bias, resid, out, odt, stats, B, H, W, Cin, Cout, k, cout_valid, bn = args[:15]
        h = ctypes.c_void_p()
        rc = self.L.pdae_conv_tc2_create(ctypes.byref(h), self._resolve(x), self._resolve(w), self._resolve(bias),
                                         self._resolve(resid), self._resolve(out), odt, self._resolve(stats), B, H, W, Cin,
                                         Cout, k, cout_valid, bn)
        _native.check(rc, "pdae_conv_tc2_create")
        self._tc2_handles.append(h)
        if fuse is not None:
            _native.check(self.L.pdae_conv_tc2_set_head_fuse(h, self._resolve(fuse)), "pdae_conv_tc2_set_head_fuse")
        return (self.L.pdae_conv_tc2_run, [h, None], 1, "conv_tc2")

    def _compile_tc2_skip(self, args):
        x, w, bias, x2, w2, Cin2, out, odt, stats, B, H, W, Cin, Cout, k, bn = args
        h = ctypes.c_void_p()
        if isinstance(x2, tuple):   # skip input = virtual concat of two tensors
            xa, Ca, xb, Cb = x2
            rc = self.L.pdae_conv_tc2_create_skip2(ctypes.byref(h), self._resolve(x), self._resolve(w), self._resolve(bias),
                                                   self._resolve(xa), Ca, self._resolve(xb), Cb, self._resolve(w2),
                                                   self._resolve(out), odt, self._resolve(stats), B, H, W, Cin, Cout, k, bn)
            _native.check(rc, "pdae_conv_tc2_create_skip2")
            self._tc2_handles.append(h)
            return (self.L.pdae_conv_tc2_run, [h, None], 1, "conv_tc2")
        rc = self.L.pdae_conv_tc2_create_skip(ctypes.byref(h), self._resolve(x), self._resolve(w), self._resolve(bias),
                                              self._resolve(x2), self._resolve(w2), Cin2, self._resolve(out), odt,
                                              self._resolve(stats), B, H, W, Cin, Cout, k, bn)
        _native.check(rc, "pdae_conv_tc2_create_skip")
        self._tc2_handles.append(h)
        return (self.L.pdae_conv_tc2_run, [h, None], 1, "conv_tc2")

    def _compile_tc3(self, args):
        (s1, C1, s2, C2, sdt, ab, silu, w, bias, k1, S1, k2, S2, wsk, resid, out, odt, stats, B, H, W, Cout, bn) = args
        h = ctypes.c_void_p()
        rc = self.L.pdae_conv_tc3_create(ctypes.byref(h), self._resolve(s1), C1, self._resolve(s2), C2, sdt, self._resolve(ab), silu,
                                         self._resolve(w), self._resolve(bias), self._resolve(k1), S1, self._resolve(k2), S2,
                                         self._resolve(wsk), self._resolve(resid), self._resolve(out), odt, self._resolve(stats),
                                         B, H, W, Cout, bn)
        _native.check(rc, "pdae_conv_tc3_create")
        self._tc3_handles.append(h)
        return (self.L.pdae_conv_tc3_run, [h, None], 1, "conv_tc3")

    def _compile_wgrad(self, args, split: bool):
        act, dy, dw, B, H, W, Cin, Cout, k = args
        h = ctypes.c_void_p()
        create = self.L.pdae_wgrad_tc_create if split else self.L.pdae_wgrad_tc_create_bf16
        rc = create(ctypes.byref(h), self._resolve(act), self._resolve(dy), self._resolve(dw), B, H, W, Cin, Cout, k)
        _native.check(rc, create.__name__)
        self._wg_handles.append(h)
        return (self.L.pdae_wgrad_tc_run, [h, None], 1, "wgrad_tc" if split else "wgrad_tc_bf16")

    def _compile_s2(self, fn, args):
        """3x3 stride-2 convs: forward (a = bf16 or split-operand input, b = [9][Cout][Cin] weights, c = fp32 or bf16 output,
        optional statistics), data gradient (a = bf16 dy, b = [9][Cin][Cout] weights, c = fp32 dx), weight gradient
        (a = bf16 input, b = bf16 dy, c = fp32 dw).  H, W: the conv's input size."""
        h = ctypes.c_void_p()
        if fn == "conv_tc2_s2":
            a, b, bias, c, odt, stats, B, H, W, Cin, Cout = args
            create = self.L.pdae_conv_tc2_create_s2_ex
            rc = create(ctypes.byref(h), self._resolve(a), self._resolve(b), self._resolve(bias), self._resolve(c), odt,
                        self._resolve(stats), B, H, W, Cin, Cout)
        else:
            a, b, c, B, H, W, Cin, Cout = args
            create = self.L.pdae_conv_tc2_create_s2_dgrad if fn == "conv_tc2_s2_dgrad" else self.L.pdae_wgrad_tc_create_bf16_s2
            rc = create(ctypes.byref(h), self._resolve(a), self._resolve(b), self._resolve(c), B, H, W, Cin, Cout)
        _native.check(rc, create.__name__)
        if fn == "wgrad_tc_bf16_s2":
            self._wg_handles.append(h)
            return (self.L.pdae_wgrad_tc_run, [h, None], 1, fn)
        self._tc2_handles.append(h)
        return (self.L.pdae_conv_tc2_run, [h, None], 1, fn)

    def _compile_splitk(self, args):
        x, w, bias, out, B, Cin, Cout = args
        h = ctypes.c_void_p()
        rc = self.L.pdae_conv_tc2_create_splitk(ctypes.byref(h), self._resolve(x), self._resolve(w), self._resolve(bias),
                                                self._resolve(out), B, Cin, Cout)
        _native.check(rc, "pdae_conv_tc2_create_splitk")
        self._tc2_handles.append(h)
        return (self.L.pdae_conv_tc2_run, [h, None], 1, "conv_tc2_splitk")

    def _compile_gemm_softmax(self, args):
        a, a_ld, a_bs, b, b_ld, b_bs, out, o_ld, o_bs, batch, M, N, K, alpha = args
        h = ctypes.c_void_p()
        rc = self.L.pdae_gemm_tc2_softmax_create(ctypes.byref(h), self._resolve(a), a_ld, a_bs, self._resolve(b), b_ld, b_bs,
                                                 self._resolve(out), o_ld, o_bs, batch, M, N, K, alpha)
        _native.check(rc, "pdae_gemm_tc2_softmax_create")
        self._tc2_handles.append(h)
        return (self.L.pdae_conv_tc2_run, [h, None], 1, "gemm_tc2")

    def _compile_gemm_major(self, args):
        a, a_mn, a_ld, a_bs, b, b_mn, b_ld, b_bs, out, o_ld, o_bs, batch, M, N, K = args
        h = ctypes.c_void_p()
        rc = self.L.pdae_gemm_tc2_create_major(ctypes.byref(h), self._resolve(a), a_mn, a_ld, a_bs, self._resolve(b), b_mn, b_ld,
                                               b_bs, self._resolve(out), o_ld, o_bs, batch, M, N, K)
        _native.check(rc, "pdae_gemm_tc2_create_major")
        self._tc2_handles.append(h)
        return (self.L.pdae_conv_tc2_run, [h, None], 1, "gemm_tc2_major")

    def _compile_gemm_softmax_grad(self, args):
        a, a_ld, a_bs, b, b_ld, b_bs, pr, p_ld, p_bs, out, o_ld, o_bs, batch, M, N, K, alpha = args
        h = ctypes.c_void_p()
        rc = self.L.pdae_gemm_tc2_softmax_grad_create(ctypes.byref(h), self._resolve(a), a_ld, a_bs, self._resolve(b), b_ld, b_bs,
                                                      self._resolve(pr), p_ld, p_bs, self._resolve(out), o_ld, o_bs, batch, M, N,
                                                      K, alpha)
        _native.check(rc, "pdae_gemm_tc2_softmax_grad_create")
        self._tc2_handles.append(h)
        return (self.L.pdae_conv_tc2_run, [h, None], 1, "gemm_tc2_softmax_grad")

    def _compile_gemm(self, args):
        a, a_ld, a_bs, b, b_ld, b_bs, out, odt, o_ld, o_bs, batch, M, N, K = args
        h = ctypes.c_void_p()
        rc = self.L.pdae_gemm_tc2_create(ctypes.byref(h), self._resolve(a), a_ld, a_bs, self._resolve(b), b_ld, b_bs,
                                         self._resolve(out), odt, o_ld, o_bs, batch, M, N, K)
        _native.check(rc, "pdae_gemm_tc2_create")
        self._tc2_handles.append(h)
        return (self.L.pdae_conv_tc2_run, [h, None], 1, "gemm_tc2")

    def gemm_tc(self, a, a_ld, a_bs, b, b_ld, b_bs, out, out_ld, out_bs, *, batch, M, N, K, out_dtype,
                softmax_alpha: Optional[float] = None, flops: Optional[float] = None, a_mn: bool = False, b_mn: bool = False,
                softmax_grad: Optional[tuple] = None) -> None:
        """Batched out_i = A_i (MxK) * B_i (NxK)^T on the persistent wgmma kernel; a/b/out are Buf or BufView.
        softmax_alpha: store softmax_rows(alpha * out_i) (bf16) instead -- needs N in {64,128,256} (row inside one tile).
        a_mn / b_mn: that operand is stored MN-major, A_i as [K][M] / B_i as [K][N] with *_ld elements between k rows (fp32 out).
        softmax_grad = (P, p_ld, p_bs, alpha): store alpha * P_i * (out_i - rowsum(P_i * out_i)) (bf16) instead, P_i being bf16
        with the output's shape -- the attention backward's dS; K-major operands, N in {64,128,256}."""
        if softmax_grad is not None:
            pr, p_ld, p_bs, alpha = softmax_grad
            assert out_dtype == torch.bfloat16 and N in (64, 128, 256) and softmax_alpha is None and not (a_mn or b_mn)
            self.call("gemm_tc2_softmax_grad", a, a_ld, a_bs, b, b_ld, b_bs, pr, p_ld, p_bs, out, out_ld, out_bs, batch, M, N, K,
                      ctypes.c_float(alpha), flops=2.0 * batch * M * N * K)
            return
        if a_mn or b_mn:
            assert out_dtype == torch.float32 and softmax_alpha is None
            self.call("gemm_tc2_major", a, int(a_mn), a_ld, a_bs, b, int(b_mn), b_ld, b_bs, out, out_ld, out_bs, batch, M, N, K,
                      flops=2.0 * batch * M * N * K if flops is None else flops)
            return
        if softmax_alpha is not None:
            assert out_dtype == torch.bfloat16 and N in (64, 128, 256)
            self.call("gemm_tc2_softmax", a, a_ld, a_bs, b, b_ld, b_bs, out, out_ld, out_bs, batch, M, N, K,
                      ctypes.c_float(softmax_alpha), flops=2.0 * batch * M * N * K)
            return
        self.call("gemm_tc2", a, a_ld, a_bs, b, b_ld, b_bs, out, _DT[out_dtype], out_ld, out_bs, batch, M, N, K,
                  flops=2.0 * batch * M * N * K if flops is None else flops)

    def can_gemm_tc(self, M: int, N: int, K: int) -> bool:
        return self.tc and not self.x3 and M % 128 == 0 and N % 64 == 0 and K % 64 == 0

    def can_gemm_x3(self, M: int, N: int, K: int) -> bool:
        """Batched GEMM in the split-operand mode: K is the LOGICAL depth (the operand blocks hold 3*K)."""
        return self.x3 and M % 128 == 0 and N % 64 == 0 and K % 64 == 0

    def __del__(self):
        try:
            for h in self._tc2_handles:
                self.L.pdae_conv_tc2_destroy(h)
            for h in self._tc3_handles:
                self.L.pdae_conv_tc3_destroy(h)
            for h in self._wg_handles:
                self.L.pdae_wgrad_tc_destroy(h)
            for h in self._nplan_handles:
                self.L.pdae_plan_destroy(h)
        except Exception:
            pass

    # ---- execution --------------------------------------------------------------------------
    def stale(self) -> bool:
        return any(p.data_ptr() != ptr for p, ptr in self.params)

    def _build_native(self, idx: List[int]):
        """Record the compiled ops `idx` into a native launch plan (include/pdae_b200.h: pdae_plan_*)."""
        if not idx:
            return None
        h = ctypes.c_void_p()
        _native.check(self.L.pdae_plan_create(ctypes.byref(h)), "pdae_plan_create")
        self._nplan_handles.append(h)
        for i in idx:
            cfn, cargs, sidx, name = self._compiled[i]
            blob = _native.pack_args(cfn, cargs)
            _native.check(self.L.pdae_plan_add(h, cfn.__name__.encode(), blob, len(cargs), sidx), "pdae_plan_add(" + cfn.__name__ + ")")
        return h

    def _launch_all(self, idx: Optional[List[int]] = None) -> None:
        stream = ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        if self._native_plans and (idx is None or idx is self._pro_idx):
            h = self._native_plans["main" if idx is None else "pro"]
            if h is not None:
                _native.check(self.L.pdae_plan_run_step(h, stream), "pdae_plan_run_step")
            return
        for i in (self._main_idx if idx is None else idx):
            cfn, cargs, sidx, name = self._compiled[i]
            cargs[sidx] = stream
            rc = cfn(*cargs)
            if rc != 0:
                _native.check(rc, "pdae_" + name)

    def refresh_packed(self, force: bool = False) -> None:
        for pk in self.packed:
            pk.refresh(force)

    def run_prologue(self) -> None:
        """Launch only the step-invariant ops (after the loop's constant inputs have been written).  Called once per
        sampling loop: the packed weight copies are re-derived unconditionally here (cost: one pass over the weights per
        ~100 network evaluations), so weights updated through `.data` / raw pointers are never stale in a loop."""
        self.refresh_packed(force=True)
        if self._pro_idx:
            self._launch_all(self._pro_idx)

    def run(self, prologue: bool = True) -> None:
        for pk in self.packed:
            pk.refresh()
        if prologue and self._pro_idx:
            self._launch_all(self._pro_idx)
        if self.graph is not None:
            self.graph.replay()
        else:
            self._launch_all()

    def capture_graph(self) -> "Plan":
        """Record the whole launch list into a CUDA graph (all buffers are static, nothing allocates), so a replay costs
        one launch instead of hundreds of ctypes calls.  Idempotent."""
        if self.graph is not None:
            return self
        self.refresh_packed(force=True)
        self._launch_all(self._pro_idx)
        self._launch_all()  # warm-up outside capture (lazy module loading, cudaFuncSetAttribute, ...)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._launch_all()
        self.graph = g
        return self

    def profile(self, reps: int = 3) -> Dict[str, Dict[str, float]]:
        """Per-kernel-kind device time (CUDA events on the launching stream) and algorithmic FLOPs of one replay.
        Measurement aid for bench.py / profiles; not used on the product path."""
        for pk in self.packed:
            pk.refresh()
        st = torch.cuda.current_stream(self.device)
        stream = ctypes.c_void_p(st.cuda_stream)
        n = len(self._compiled)
        acc = [0.0] * n
        self._launch_all(self._pro_idx)
        for _ in range(reps):
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(self._main_idx) + 1)]
            evs[0].record(st)
            for k, i in enumerate(self._main_idx):
                cfn, cargs, sidx, name = self._compiled[i]
                cargs[sidx] = stream
                _native.check(cfn(*cargs), "pdae_" + name)
                evs[k + 1].record(st)
            st.synchronize()
            for k, i in enumerate(self._main_idx):
                acc[i] += evs[k].elapsed_time(evs[k + 1]) / reps
        self.last_op_ms = acc  # per recorded op, same order as self.ops (0 for prologue ops: not part of a step)
        out: Dict[str, Dict[str, float]] = {}
        for i in self._main_idx:
            name = self._compiled[i][3]
            d = out.setdefault(name, {"ms": 0.0, "flops": 0.0, "launches": 0})
            d["ms"] += acc[i]
            d["flops"] += self.flops[i]
            d["launches"] += 1
        return out

    # ---- emitters: thin typed wrappers that pick kernels ------------------------------------------
    def use_tc(self, Cin: int, Cout: int, k: int, stride: int, H: int, W: int) -> bool:
        return self.tc and self._tc_shape_ok(Cin, Cout, k, stride, H, W)

    def can_conv_s2(self, H: int, W: int, Cin: int, Cout: int) -> bool:
        """Does a forward-only plan run a 3x3 stride-2 pad-1 conv of an H x W input on the tensor cores (Plan.conv, with a bf16
        or split-operand input)?  Training forward plans keep their own rules (train_tc)."""
        return self.tc and self.train_tc is None and bool(self.L.pdae_conv_s2_tc_supported(H, W, Cin, Cout))

    def _tc_shape_ok(self, Cin: int, Cout: int, k: int, stride: int, H: int, W: int) -> bool:
        if stride != 1 or k not in (1, 3) or Cin % 64 or Cout % 64:
            return False
        tw = 1
        while tw * 2 <= 128 and W % (tw * 2) == 0:
            tw *= 2
        th = 1
        while th * 2 <= 128 // tw and H % (th * 2) == 0:
            th *= 2
        return W % tw == 0 and H % th == 0 and 128 % (tw * th) == 0

    def conv(self, x: Buf, weight: torch.Tensor, bias: Optional[torch.Tensor], out: Buf, *, B, H, W, Cin, Cout, k=3,
             stride=1, pad=None, residual: Optional[Buf] = None, in_nchw=False, out_nchw=False, a_silu=False,
             wkey=None, want_stats=False, bn_override=0, skip=None, w_transform=None) -> Optional[Buf]:
        """weight: nn-style [Cout, Cin, k, k] / [Cout, Cin, 1] / [Cout, Cin] parameter.
        w_transform (tensor-core path only): maps the detached parameter to the [Cout, Cin, k, k] tensor actually convolved
        with (e.g. the transposed, flipped weights of a dgrad) -- the packed copy still tracks the PARAMETER's version.
        Returns the per-channel (sum, sum^2) buffer [B][Cout][2] if the tensor-core epilogue produced one."""
        pad = k // 2 if pad is None else pad
        if (self.train_tc == "bf16" and x.dtype == torch.bfloat16 and not (in_nchw or out_nchw or a_silu) and skip is None
                and w_transform is None and pad == k // 2 and self._tc_shape_ok(Cin, Cout, k, stride, H, W)):
            # an input that is already a plain bf16 tensor in a bf16 training forward (the attention block's normalised input and
            # attention output): conv_tc2 reads it as it is, and it is its own copy for the backward's weight gradient
            wp = self.pack((wkey or id(weight), "tc"), [weight],
                           lambda: weight.detach().reshape(Cout, Cin, k * k).permute(2, 0, 1).to(torch.bfloat16))
            x.tc_copy = x
            self.call("conv_tc2", x, wp, self.param(bias), residual, out, _DT[out.dtype], None, B, H, W, Cin, Cout, k, 0,
                      bn_override, flops=2.0 * B * H * W * Cout * Cin * k * k)
            return None
        if (self.train_tc == "bf16" and stride == 2 and k == 3 and pad == 1 and x.dtype == torch.float32
                and out.dtype == torch.float32 and not (in_nchw or out_nchw or a_silu) and skip is None and w_transform is None
                and residual is None and self.L.pdae_conv_s2_tc_supported(H, W, Cin, Cout)):
            # 3x3 stride-2 conv of a bf16 training forward (the semantic encoder under autocast): conv_tc2 reads a plain bf16
            # copy of the input through its parity view; the backward's weight gradient reads the same copy
            xt = self.new((B, H, W, Cin), torch.bfloat16, "train_bf16")
            self.call("gn_apply", x, PDAE_F32, Cin, None, PDAE_F32, 0, None, 0, RESAMPLE_NONE, B, H, W, xt, PDAE_BF16, None,
                      PDAE_F32, _STREAM)
            wp = self.pack((wkey or id(weight), "tc"), [weight],
                           lambda: weight.detach().reshape(Cout, Cin, 9).permute(2, 0, 1).to(torch.bfloat16))
            x.tc_copy = xt
            self.call("conv_tc2_s2", xt, wp, self.param(bias), out, PDAE_F32, None, B, H, W, Cin, Cout,
                      flops=2.0 * B * (H // 2) * (W // 2) * Cout * Cin * 9)
            return None
        if (self.train_tc is None and stride == 2 and k == 3 and pad == 1 and x.dtype == torch.bfloat16
                and not (in_nchw or out_nchw or a_silu) and skip is None and w_transform is None and residual is None
                and self.can_conv_s2(H, W, Cin, Cout)):
            # forward-only 3x3 stride-2 conv in a tensor-core mode (the semantic encoder): conv_tc2 reads the bf16 activation
            # ("bf16") or its [hi | lo | hi] split copy ("bf16x3") through its parity view; the epilogue writes the output in its
            # dtype and, on request, the per-channel statistics of the stored values
            if x.split3:
                wp = self.pack((wkey or id(weight), "tc_x3"), [weight],
                               lambda Cin=Cin: split3_weights(weight.detach().reshape(Cout, Cin, 9)))
            else:
                wp = self.pack((wkey or id(weight), "tc"), [weight],
                               lambda: weight.detach().reshape(Cout, Cin, 9).permute(2, 0, 1).to(torch.bfloat16))
            stats = self.new_stats(B, Cout) if want_stats else None
            self.call("conv_tc2_s2", x, wp, self.param(bias), out, _DT[out.dtype], stats, B, H, W, 3 * Cin if x.split3 else Cin,
                      Cout, flops=2.0 * B * (H // 2) * (W // 2) * Cout * Cin * 9)
            return stats
        if (self.train_tc and x.dtype == torch.float32 and out.dtype == torch.float32 and not (in_nchw or out_nchw or a_silu)
                and skip is None and w_transform is None and pad == k // 2 and self._tc_shape_ok(Cin, Cout, k, stride, H, W)):
            if self.train_tc == "bf16x3":
                xt = self.new((B, H, W, 3 * Cin), torch.bfloat16, "train_split3")
                xt.split3 = True
                self.call("gn_apply_split3", x, Cin, None, 0, None, 0, RESAMPLE_NONE, B, H, W, xt, None, PDAE_F32, _STREAM)
                wp = self.pack((wkey or id(weight), "tc_x3"), [weight],
                               lambda Cin=Cin: split3_weights(weight.detach().reshape(Cout, Cin, k * k)))
                Ce = 3 * Cin
            elif self.train_tc == "bf16":
                xt = self.new((B, H, W, Cin), torch.bfloat16, "train_bf16")
                self.call("gn_apply", x, PDAE_F32, Cin, None, PDAE_F32, 0, None, 0, RESAMPLE_NONE, B, H, W, xt, PDAE_BF16, None,
                          PDAE_F32, _STREAM)
                wp = self.pack((wkey or id(weight), "tc"), [weight],
                               lambda: weight.detach().reshape(Cout, Cin, k * k).permute(2, 0, 1).to(torch.bfloat16))
                Ce = Cin
            else:
                raise ValueError(f"Plan.train_tc must be None, 'bf16x3' or 'bf16', not {self.train_tc!r}")
            x.tc_copy = xt      # the backward's tensor-core weight gradient reads the same bf16 activation
            self.call("conv_tc2", xt, wp, self.param(bias), residual, out, PDAE_F32, None, B, H, W, Ce, Cout, k, 0,
                      bn_override, flops=2.0 * B * H * W * Cout * Cin * k * k)
            return None
        bias_b = self.param(bias)
        wkey = wkey or id(weight)
        if x.dtype == torch.bfloat16 and self.use_tc(Cin, Cout, k, stride, H, W) and not (in_nchw or out_nchw or a_silu):
            x3 = bool(x.split3)
            fl = 2.0 * B * H * W * Cout * Cin * k * k     # algorithmic (the x3 mode issues 3x the MMAs for it)
            wsrc = (lambda: w_transform(weight.detach())) if w_transform is not None else (lambda: weight.detach())
            if x3:   # activation blocks [a_hi | a_lo | a_hi] x weight blocks [W_hi | W_hi | W_lo]
                wp = self.pack((wkey, "tc_x3"), [weight], lambda Cin=Cin: split3_weights(wsrc().reshape(Cout, Cin, k * k)))
                Cin = 3 * Cin
            else:
                wp = self.pack((wkey, "tc"), [weight],
                               lambda: wsrc().reshape(Cout, Cin, k * k).permute(2, 0, 1).to(torch.bfloat16))
            stats = self.new_stats(B, Cout) if want_stats else None
            if skip is not None:
                # fused 1x1 skip conv (model/module.py:268-276): extra K blocks accumulated into the same accumulator tile
                sk_in, sw, sb, Cin2 = skip   # sk_in: a bf16 buffer, or (buf_a, Ca, buf_b, Cb) = their channel concat
                assert residual is None
                if isinstance(sk_in, tuple):
                    assert sk_in[0].dtype == sk_in[2].dtype == torch.bfloat16 and sk_in[1] + sk_in[3] == Cin2 and not x3
                else:
                    assert sk_in.dtype == torch.bfloat16 and bool(sk_in.split3) == x3
                if x3:
                    w2 = self.pack((id(sw), "tc_skip_x3"), [sw],
                                   lambda Cin2=Cin2: split3_weights(sw.detach().reshape(Cout, Cin2, 1))[0])   # (bind the logical Cin2: it is tripled below, and this runs again on every weight refresh)
                    Cin2 = 3 * Cin2
                else:
                    w2 = self.pack((id(sw), "tc_skip"), [sw], lambda: sw.detach().reshape(Cout, Cin2).to(torch.bfloat16))
                bsum = self.pack((id(bias), id(sb), "bias_sum"), [bias, sb], lambda: (bias.detach() + sb.detach()).float())
                self.params.append((sb, sb.data_ptr()))
                self.call("conv_tc2_skip", x, wp, bsum, sk_in, w2, Cin2, out, _DT[out.dtype], stats, B, H, W, Cin, Cout, k,
                          bn_override, flops=fl + 2.0 * B * H * W * Cout * (Cin2 // 3 if x3 else Cin2))
                return stats
            self.call("conv_tc2", x, wp, bias_b, residual, out, _DT[out.dtype], stats, B, H, W, Cin, Cout, k, 0,
                      bn_override, flops=fl)
            return stats
        assert out.dtype == torch.float32, "CUDA-core conv writes fp32"
        wp = self.pack((wkey, "simt"), [weight], lambda: weight.detach().reshape(Cout, Cin, k * k).permute(2, 1, 0).float())
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        self.call("conv2d_simt", x, _DT[x.dtype], int(in_nchw), wp, bias_b, residual, out, int(out_nchw), B, H, W, Cin, Cout,
                  k, stride, pad, int(a_silu), _STREAM, flops=2.0 * B * Ho * Wo * Cout * Cin * k * k)
        return None

    # ---- fused-prologue conv (conv_tc3) --------------------------------------------------------------------------------
    def can_fuse_prologue(self, srcs: Sequence[Tuple[Optional[Buf], int]], Cout: int, H: int, W: int) -> bool:
        """3x3 stride-1 conv whose input is SiLU(a*x+b) of (a virtual concat of) NHWC tensors already in this mode's
        stream dtype: 16 x 8 output tiles of one image, 64-channel k-blocks that do not straddle the concat seam."""
        if not self.tc or H % 16 or W % 8 or Cout % 64:
            return False
        want = torch.float32 if self.x3 else torch.bfloat16
        for b, C in srcs:
            if b is None:
                continue
            if C <= 0 or C % 64 or b.dtype != want or b.split3:
                return False
        return True

    def coef_buffer(self, ab) -> Buf:
        """Materialise deferred GroupNorm coefficients ([B][2][C] fp32: a | b) with one gn_coef_ch launch."""
        if not isinstance(ab, CoefSpec):
            return ab
        c = ab
        buf = self.new((c.B, 2, c.C1 + c.C2), torch.float32, "gn_ab")
        self.call("gn_coef_ch", c.stats1, c.C1, c.stats2, c.C2, c.gamma, c.beta, c.B, c.HW, ctypes.c_float(1e-5),
                  c.emb, c.emb_ld, c.embz, c.embz_ld, buf, _STREAM)
        return buf

    def conv_fused(self, s1: Buf, C1: int, s2: Optional[Buf], C2: int, ab, weight: torch.Tensor, bias: Optional[torch.Tensor],
                   out: Buf, *, B, H, W, Cout, silu=True, residual: Optional[Buf] = None, skip=None, want_stats=False,
                   bn_override=0) -> Optional["BufView"]:
        """out = conv3x3(SiLU(a*cat(s1, s2)+b)) + bias (+ residual | + 1x1 skip conv of cat(skip sources)) on conv_tc3.
        skip = (k1, S1, k2, S2, skip_weight, skip_bias): raw (un-normalised) sources of the ResBlock's skip_connection."""
        Cin = C1 + C2
        x3 = self.x3
        ab = self.coef_buffer(ab)
        if x3:
            def pack3(Cin=Cin):
                w = weight.detach().reshape(Cout, Cin, 9).float()
                hi = w.to(torch.bfloat16)
                lo = (w - hi.float()).to(torch.bfloat16)
                return torch.stack([hi, lo], 0).permute(3, 0, 1, 2).contiguous()          # [9][2][Cout][Cin]
            wp = self.pack((id(weight), "tc3_x3"), [weight], pack3)
        else:
            wp = self.pack((id(weight), "tc"), [weight],
                           lambda: weight.detach().reshape(Cout, Cin, 9).permute(2, 0, 1).to(torch.bfloat16))
        fl = 2.0 * B * H * W * Cout * Cin * 9
        k1 = k2 = wsk = None
        S1 = S2 = 0
        if skip is not None:
            assert residual is None
            k1, S1, k2, S2, sw, sb = skip
            Cs = S1 + S2
            if x3:
                def packs(Cs=Cs):
                    w = sw.detach().reshape(Cout, Cs).float()
                    hi = w.to(torch.bfloat16)
                    return torch.stack([hi, (w - hi.float()).to(torch.bfloat16)], 0).contiguous()   # [2][Cout][Cs]
                wsk = self.pack((id(sw), "tc3_skip_x3"), [sw], packs)
            else:
                wsk = self.pack((id(sw), "tc_skip"), [sw], lambda: sw.detach().reshape(Cout, Cs).to(torch.bfloat16))
            bias_b = self.pack((id(bias), id(sb), "bias_sum"), [bias, sb], lambda: (bias.detach() + sb.detach()).float())
            self.params.append((sb, sb.data_ptr()))
            self.params.append((bias, bias.data_ptr()))
            fl += 2.0 * B * H * W * Cout * Cs
        else:
            bias_b = self.param(bias)
        stats = self.new_stats(B, Cout) if want_stats else None
        self.call("conv_tc3", s1, C1, s2, C2, PDAE_F32 if x3 else PDAE_BF16, ab, int(silu), wp, bias_b, k1, S1, k2, S2, wsk,
                  residual, out, _DT[out.dtype], stats, B, H, W, Cout, bn_override, flops=fl)
        return stats

    def linear(self, x: Buf, weight: torch.Tensor, bias: Optional[torch.Tensor], out: Buf, *, B, Cin, Cout, a_silu=False,
               wkey=None) -> None:
        self.conv(x, weight, bias, out, B=B, H=1, W=1, Cin=Cin, Cout=Cout, k=1, a_silu=a_silu, wkey=wkey)

    def linear_packed(self, x: Buf, wp: Buf, bias: Optional[Buf], out: Buf, *, B, Cin, Cout, a_silu=False) -> None:
        """Linear with an already packed fp32 [Cin][Cout] weight (e.g. all blocks' emb layers concatenated)."""
        self.call("conv2d_simt", x, PDAE_F32, 0, wp, bias, None, out, 0, B, 1, 1, Cin, Cout, 1, 1, 0, int(a_silu), _STREAM,
                  flops=2.0 * B * Cin * Cout)

    def linear_tc(self, x, wp: Buf, bias: Optional[Buf], *, B, Cin, Cout, name="linear_tc", out: Optional[Buf] = None,
                  flops: Optional[float] = None):
        """out[B][Cout] (fp32) = x[B][Cin] (bf16) wp[Cout][Cin]^T (bf16) + bias, one bf16 MMA per product on conv_tc2; returns
        out.  When the output tiles alone would leave SMs idle (the latent MLP's Linears at training batch sizes: one 128-row
        tile row) it runs split-K (pdae_conv_tc2_create_splitk): out is then a slice of the plan's zeroed arena, which the
        plan's leading pdae_zero op clears on every replay, and the partial tiles are added into it.
        out: a given fp32 [B][Cout] buffer (e.g. a plan output) to write instead; under split-K a pdae_zero op clears it first.
        flops: the algorithmic FLOPs to record (a split-operand x / wp hold three bf16 blocks per logical channel)."""
        assert Cin % 64 == 0 and Cout % 64 == 0, (Cin, Cout)
        fl = 2.0 * B * Cin * Cout if flops is None else flops
        if self.det:
            # deterministic split-K at every batch size: its k ranges follow Cin and Cout alone, so a row's bits do not depend
            # on how many rows the GEMM has (the latent loop's one-row bank GEMM equals the B-row one); no zeroing needed
            if out is None:
                out = self.new((B, Cout), torch.float32, name)
            self.call("conv_tc2_splitk", x, wp, bias, out, B, Cin, Cout, flops=fl)
            return out
        tiles = -(-B // 128) * (Cout // (128 if Cout % 128 == 0 else 64))   # = conv_tc2's output tiles
        if tiles < torch.cuda.get_device_properties(self.device).multi_processor_count:
            if out is None:
                out = self.new_zeroed(B * Cout)
            else:
                self.call("zero", out, ctypes.c_int64(B * Cout * 4), _STREAM)
            self.call("conv_tc2_splitk", x, wp, bias, out, B, Cin, Cout, flops=fl)
            return out
        if out is None:
            out = self.new((B, Cout), torch.float32, name)
        self.call("conv_tc2", x, wp, bias, None, out, PDAE_F32, None, B, 1, 1, Cin, Cout, 1, 0, 0, flops=fl)
        return out

    def head_conv(self, x: Buf, weight: torch.Tensor, bias: torch.Tensor, out_nchw: Buf, *, B, H, W, Cin, Cout,
                  fuse_key: Optional[str] = None) -> None:
        """3x3 conv to a few image channels (unet.py:171-175).  fuse_key ("eps" | "grad"): on the tensor-core head, reserve a
        device-side descriptor through which a sampling loop can switch on the DDIM update fused into this head's epilogue
        (Plan.head_fuse[fuse_key]; all-zero = plain head)."""
        fl = 2.0 * B * H * W * Cout * Cin * 9
        if x.dtype == torch.bfloat16 and Cout <= 16 and self.use_tc(Cin, 64, 3, 1, H, W):
            # tensor-core head: Cout zero-padded to one 16-wide UMMA tile, NCHW fp32 planes written by the epilogue
            x3 = bool(x.split3)
            Ce = 3 * Cin if x3 else Cin

            def pack16():
                w = weight.detach().reshape(Cout, Cin, 9)
                w = split3_weights(w) if x3 else w.permute(2, 0, 1).to(torch.bfloat16)     # [9][Cout][Ce]
                z = torch.zeros(9, 16, Ce, device=w.device, dtype=torch.bfloat16)
                z[:, :Cout, :] = w
                return z
            wp = self.pack((id(weight), "tc16_x3" if x3 else "tc16"), [weight], pack16)
            fuse = None
            if fuse_key is not None:
                with torch.inference_mode(False):
                    fuse = self.fixed(torch.zeros(FUSE_DESC_LEN, dtype=torch.int64, device=self.device))
                self.head_fuse[fuse_key] = fuse
            self.call("conv_tc2", x, wp, self.param(bias), None, out_nchw, PDAE_F32, None, B, H, W, Ce, 16, 3, Cout, 0, fuse, flops=fl)
        elif Cout <= 4 and Cin % 4 == 0:
            assert x.dtype in (torch.float32, torch.bfloat16)

            def pack4():
                w = weight.detach().reshape(Cout, Cin, 9).permute(2, 1, 0).float()
                z = torch.zeros(9, Cin, 4, device=w.device, dtype=torch.float32)
                z[:, :, :Cout] = w
                return z
            wp = self.pack((id(weight), "small4"), [weight], pack4)
            self.call("conv3x3_smalln", x, _DT[x.dtype], wp, self.param(bias), out_nchw, B, H, W, Cin, Cout, _STREAM, flops=fl)
        else:
            assert x.dtype == torch.float32
            self.conv(x, weight, bias, out_nchw, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=3, out_nchw=True)

    def head_act_dtype(self, Cin: int, Cout: int, H: int, W: int):
        """dtype the normalised input of an image-head conv should be produced in (bf16 only if a bf16 kernel takes it)."""
        if not self.tc:
            return torch.float32
        if Cout <= 16 and self.use_tc(Cin, 64, 3, 1, H, W):
            return torch.bfloat16
        if Cout <= 4 and Cin % 4 == 0 and not self.x3:      # CUDA-core small-N head: plain bf16 input (fp32 in the x3 mode)
            return torch.bfloat16
        return torch.float32

    def new_stats(self, B: int, C: int):
        """A [B][C][2] fp32 accumulator inside the plan's statistics arena (ONE memset per replay zeroes them all).  A
        deterministic plan's kernels write their statistics instead of adding them: a plain arena buffer, no memset."""
        if self.det:
            return self.new((B, C, 2), torch.float32, "chs")
        off = self._stats_elems
        self._stats_elems += B * C * 2
        return BufView(self._stats_arena, off)

    def ch_stats(self, src: Buf, C: int, *, B, HW) -> Buf:
        """Per-channel (sum, sum^2) of an fp32 NHWC tensor that no conv epilogue produced."""
        chs = self.new((B, C, 2), torch.float32, "chs")
        if self.det:
            ws = self._det_workspace(B, HW, C)
            self.call("ch_stats_det", src, B, HW, C, chs, ws, ctypes.c_int64(ws.nbytes), _STREAM)
            return chs
        self.call("ch_stats", src, B, HW, C, chs, _STREAM)
        return chs

    def _det_workspace(self, B: int, HW: int, C: int) -> Buf:
        """Arena scratch for the per-CTA slots of ch_stats_det / gn_stats_det."""
        n = int(self.L.pdae_stats_det_workspace_bytes(B, HW, C))
        _native.check(min(n, 0), "pdae_stats_det_workspace_bytes")
        return self.new((max(n, 16) // 4,), torch.float32, "stats_slots")

    def stem_conv_bf16(self, x_in: Buf, wp: Buf, bias: Optional[torch.Tensor], out: Buf, *, B, H, W, Cin, Cout, stride,
                       flops: float):
        """The CUDA-core stem (stride 1 or 2) writing the bf16 stream and the first GroupNorm's [B][Cout][2] statistics;
        returns the statistics buffer."""
        st = self.new_stats(B, Cout)
        if self.det:
            n = int(self.L.pdae_stem_conv_det_workspace_bytes(B, H, W, Cout, stride))
            _native.check(min(n, 0), "pdae_stem_conv_det_workspace_bytes")
            ws = self.new((max(n, 16) // 4,), torch.float32, "stem_slots")
            self.call("stem_conv_bf16_det", x_in, wp, self.param(bias), out, st, B, H, W, Cin, Cout, stride, ws,
                      ctypes.c_int64(ws.nbytes), _STREAM, flops=flops)
        else:
            self.call("stem_conv_bf16" if stride == 1 else "stem_conv_s2_bf16", x_in, wp, self.param(bias), out, st, B, H, W,
                      Cin, Cout, _STREAM, flops=flops)
        return st

    def stem_det_fits(self, Cin: int, Cout: int) -> bool:
        """The deterministic stem keeps its per-thread statistics in shared memory (include/pdae_b200.h)."""
        return not self.det or (9 * Cin + 2 + 2 * (256 // (Cout // 8))) * Cout * 4 <= 48 * 1024

    @property
    def fused_stats(self) -> bool:
        return self.tc

    @property
    def stream_dtype(self):
        return torch.bfloat16 if self.stream_bf16 else torch.float32

    def to_stream(self, src: Buf, C: int, *, B, H, W) -> Buf:
        """Cast an fp32 NHWC tensor into the residual-stream dtype (no-op for an fp32 stream)."""
        if not self.stream_bf16 or src.dtype == torch.bfloat16 or C % 8:
            return src
        out, _ = self.gn_apply(src, C, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W, act_dtype=torch.bfloat16)
        return out

    def gn_coef(self, src1: Buf, C1: int, src2: Optional[Buf], C2: int, gamma, beta, *, B, HW, emb=None, emb_ld=0,
                embz=None, embz_ld=0, stats1: Optional[Buf] = None, stats2: Optional[Buf] = None) -> Buf:
        """GroupNorm(32) statistics -> per-(b,c) affine coefficients.  The tensor-core modes consume the per-channel sums the
        conv epilogues accumulated (computing missing ones); fp32 mode keeps the fp64 two-kernel path."""
        C = C1 + C2
        if self.fused_stats:
            if stats1 is None:
                stats1 = self.ch_stats(src1, C1, B=B, HW=HW)
            if src2 is not None and stats2 is None:
                stats2 = self.ch_stats(src2, C2, B=B, HW=HW)
            # deferred: the consumer (gn_apply / conv_fused) launches gn_coef_ch right before the op that reads them
            return CoefSpec(stats1, C1, stats2, C2, self.param(gamma), self.param(beta), B, HW, emb, emb_ld, embz, embz_ld)
        ab = self.new((B, 2, C), torch.float32, "gn_ab")
        sums = self.new((B, 32, 2), torch.float64, "gn_sums")
        self.last_sums = sums
        if self.det:
            ws = self._det_workspace(B, HW, C)
            self.call("gn_stats_det", src1, C1, src2, C2, B, HW, sums, ws, ctypes.c_int64(ws.nbytes), _STREAM)
        else:
            self.call("gn_stats", src1, C1, src2, C2, B, HW, sums, _STREAM)
        self.call("gn_coef", sums, self.param(gamma), self.param(beta), B, C, HW, ctypes.c_float(1e-5), emb, emb_ld, embz,
                  embz_ld, ab, _STREAM)
        return ab

    def gn_apply(self, src1: Buf, C1: int, src2: Optional[Buf], C2: int, ab: Optional[Buf], *, silu: bool, resample: int,
                 B, H, W, act_dtype, raw_dtype=None) -> Tuple[Buf, Optional[Buf]]:
        C = C1 + C2
        Ho, Wo = (2 * H, 2 * W) if resample == RESAMPLE_UP2 else ((H // 2, W // 2) if resample == RESAMPLE_DOWN2 else (H, W))
        if self.x3 and act_dtype == torch.bfloat16:
            # split-operand mode: [hi | lo | hi] bf16 blocks for the tensor-core convs (fp32 sources only)
            assert src1.dtype == torch.float32 and (src2 is None or src2.dtype == torch.float32)
            if isinstance(ab, CoefSpec):
                c, ab = ab, self.new((B, 2, C), torch.float32, "gn_ab")
                self.call("gn_coef_ch", c.stats1, c.C1, c.stats2, c.C2, c.gamma, c.beta, c.B, c.HW, ctypes.c_float(1e-5),
                          c.emb, c.emb_ld, c.embz, c.embz_ld, ab, _STREAM)
            act = self.new((B, Ho, Wo, 3 * C), torch.bfloat16, "act_x3")
            act.split3 = True
            raw = None
            if raw_dtype is not None:
                raw = self.new((B, Ho, Wo, 3 * C if raw_dtype == torch.bfloat16 else C), raw_dtype, "raw_x3")
                raw.split3 = raw_dtype == torch.bfloat16
            self.call("gn_apply_split3", src1, C1, src2, C2, ab, int(silu), resample, B, H, W, act, raw,
                      _DT[raw_dtype] if raw_dtype is not None else PDAE_F32, _STREAM)
            return act, raw
        act = self.new((B, Ho, Wo, C), act_dtype, "act")
        raw = self.new((B, Ho, Wo, C), raw_dtype, "raw") if raw_dtype is not None else None
        if isinstance(ab, CoefSpec):
            c = ab
            ab = self.new((B, 2, C), torch.float32, "gn_ab")
            self.call("gn_coef_ch", c.stats1, c.C1, c.stats2, c.C2, c.gamma, c.beta, c.B, c.HW, ctypes.c_float(1e-5),
                      c.emb, c.emb_ld, c.embz, c.embz_ld, ab, _STREAM)
        self.call("gn_apply", src1, _DT[src1.dtype], C1, src2, _DT[src2.dtype] if src2 is not None else PDAE_F32, C2, ab, int(silu),
                  resample, B, H, W, act, _DT[act_dtype], raw, _DT[raw_dtype] if raw_dtype is not None else PDAE_F32, _STREAM)
        return act, raw


# Tensor-core ops a deterministic plan switches to their DET kernels at finalize (pdae_conv_tc2 / tc3 / wgrad_tc
# _set_deterministic).  The training GEMMs and the stride-2 data gradient record no statistics; their DET kernels are the same
# kernels without the compiled-in atomic statistics code (conv_tc2.cu).
DET_OPS = frozenset({"conv_tc2", "conv_tc2_skip", "conv_tc2_s2", "conv_tc2_splitk", "gemm_tc2", "gemm_tc2_softmax", "conv_tc3",
                     "gemm_tc2_major", "gemm_tc2_softmax_grad", "conv_tc2_s2_dgrad", "wgrad_tc", "wgrad_tc_bf16",
                     "wgrad_tc_bf16_s2"})


def det_entry_points(fn: str) -> Tuple[str, str]:
    """(set_deterministic, det_workspace_bytes) entry points of the handle an op of DET_OPS compiles to."""
    kind = "conv_tc3" if fn == "conv_tc3" else ("wgrad_tc" if fn.startswith("wgrad_tc") else "conv_tc2")
    return f"pdae_{kind}_set_deterministic", f"pdae_{kind}_det_workspace_bytes"


# Ops whose kernels reduce with float atomics (or accumulate into a zeroed buffer): never in a deterministic plan, whose
# recording uses the *_det ops instead.
NONDET_OPS = frozenset({"zero", "ch_stats", "gn_stats", "stem_conv_bf16", "stem_conv_s2_bf16", "conv2d_wgrad_simt",
                        "conv2d_dgrad_simt", "gn_bwd_sums", "gn_bwd_coef", "colsum", "embedding_bwd", "mlp_mod_ln_act_bwd",
                        "mlp_mod_ln_act_bwd_bf16"})

_LAUNCHES = {"gn_stats": 1, "attention_simt": 3, "zero": 0, "ch_stats_det": 2, "gn_stats_det": 2, "stem_conv_bf16_det": 2}
