"""Thin launch wrappers over the C ABI (include/b200seg.h) and the torch.autograd.Functions built from
them.  PyTorch is plumbing here: it owns device memory (caching allocator), the current stream and the
autograd tape; every FLOP and every byte of activation traffic goes through libb200seg.so.

Internal activation format: NDHWC tensors ``[B, D, H, W, ld]`` (fp16 under autocast, else fp32) plus a
side tensor of InstanceNorm sums ``stats[B, C, 2]`` (fp64) produced by whichever kernel wrote the
activation.  Channel slices of a wider tensor are addressed with (coff, C) — never with torch views —
so fused tensors (conv1+shortcut outputs, concat buffers) are consumed in place.
"""
import torch

from . import _lib
from ._lib import ACT_NONE, ACT_RELU, ALGO_AUTO, ALGO_DIRECT, ALGO_TC, ALGO_TC_TF32, F16, F32, call

IN_EPS = 1e-4  # nn.InstanceNorm3d(eps=1e-4): reference conv_layers.py:40,42


def _dt(t):
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.float32:
        return F32
    raise TypeError("b200seg supports float16/float32 activations, got %s" % t.dtype)


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _need_cuda(t):
    """Kernels launch on the CURRENT device and stream: a tensor that lives elsewhere would be an illegal address
    or a cross-stream race, so it is an error (models switch device themselves, see `on_device`)."""
    if not t.is_cuda:
        raise _lib.B200SegError("b200seg ops need CUDA tensors on an H100 — there is no CPU fallback")
    if t.device.type == "cuda" and t.device.index != torch.cuda.current_device():
        raise _lib.B200SegError("tensor lives on %s but the current CUDA device is cuda:%d — wrap the call in "
                                "torch.cuda.device(tensor.device)" % (t.device, torch.cuda.current_device()))


def on_device(t):
    """Context manager making t's device current (model.forward uses it, so DDP ranks / multi-device processes
    launch on the right GPU and the right current stream)."""
    if t.device.type != "cuda":         # CPU-emulated host-logic tests; real ops reject such tensors in _need_cuda
        import contextlib
        return contextlib.nullcontext()
    return torch.cuda.device(t.device)


def compute_dtype():
    """fp16 storage/tensor-core operands under torch.autocast (the reference's --amp path,
    train_ddp.py:181), fp32 otherwise."""
    if not torch.is_autocast_enabled():
        return torch.float32
    adt = torch.get_autocast_dtype("cuda")
    if adt != torch.float16:
        raise _lib.B200SegError("b200seg implements fp16 autocast (the reference's --amp path); autocast dtype %s is "
                                "not supported — use torch.autocast('cuda', dtype=torch.float16)" % adt)
    return torch.float16


class _ZeroArena:
    """Zero-initialised scratch (InstanceNorm sums and other accumulate-into buffers) carved out of chunks that are
    cleared with ONE memset each instead of one tiny fill kernel per buffer (161 per ResUNet step, ~1000 per MedFormer
    step in the round-2 launch lists).  A slice is handed out once and never reused; a chunk lives as long as any of its
    slices is referenced (saved for backward), so nothing is cleared twice and nothing is shared."""
    CHUNK_BYTES = 1 << 20

    def __init__(self):
        self._cur = {}          # (device, dtype) -> [chunk tensor, next free element]

    def take(self, numel, dtype, device):
        key = (str(device), dtype)
        per = 16 // torch.empty(0, dtype=dtype).element_size()           # keep every slice 16-byte aligned
        padded = (numel + per - 1) // per * per
        cur = self._cur.get(key)
        if cur is None or cur[1] + padded > cur[0].numel():
            n = max(self.CHUNK_BYTES // torch.empty(0, dtype=dtype).element_size(), padded)
            cur = [torch.zeros(n, dtype=dtype, device=device), 0]
            self._cur[key] = cur
        out = cur[0][cur[1]:cur[1] + numel]
        cur[1] += padded
        return out


_ARENA = _ZeroArena()


def zeros_scratch(shape, dtype, device):
    """A zero-filled scratch tensor from the arena (for sums a kernel accumulates into — not for tensors that are
    returned to autograd as gradients)."""
    n = 1
    for s in shape:
        n *= int(s)
    return _ARENA.take(n, dtype, device).view(*shape)


def new_stats(B, C, device):
    return zeros_scratch((B, C, 2), torch.float64, device)


# ----------------------------------------------------------------------------- raw launches
def tf32_enabled():
    """True when torch allows TF32 for fp32 matmuls (torch.backends.cuda.matmul.fp32_precision == 'tf32'), read at call
    time.  The convolutions and Linears here are implicit GEMMs, so they follow torch's matmul precision — not cuDNN's
    conv flag, which defaults to TF32 — and stay exact fp32 unless the user opts in.  Only `fp32_precision` is read:
    after the new precision API has been used, the legacy getters raise."""
    return torch.backends.cuda.matmul.fp32_precision == "tf32"


def conv_algo(Cin, Cout, ksize, dtype, B=1):
    """Algorithm (ALGO_TC / ALGO_TC_TF32 / ALGO_DIRECT) the library uses for this conv shape; also names the
    packed-weight layout.  fp32 shapes take the TF32 tensor cores only while `tf32_enabled()`."""
    lib = _lib.load()
    if dtype != torch.float16 and tf32_enabled():
        return lib.b200seg_conv3d_algo_tf32(Cin, Cout, ksize[0], ksize[1], ksize[2], B)
    return lib.b200seg_conv3d_algo(Cin, Cout, ksize[0], ksize[1], ksize[2], F16 if dtype == torch.float16 else F32, B)


_LAYOUT_CODE = {ALGO_DIRECT: 0, ALGO_TC: 1, ALGO_TC_TF32: 2}     # the job column of b200seg_pack_weights_multi


def pack_weight(w, dtype, transpose_flip=False, out=None, co_off=0, co_total=None, layout=ALGO_DIRECT):
    """[Cout,Cin,kd,kh,kw] fp32 parameter -> packed weights for `layout` (see b200seg_pack_weight)."""
    Cout, Cin = w.shape[0], w.shape[1]
    taps = w.shape[2] * w.shape[3] * w.shape[4]
    co_total = Cout if co_total is None else co_total
    if out is None:
        out = torch.empty(taps * co_total * Cin, dtype=dtype, device=w.device)
    wc = w.detach()
    if wc.dtype != torch.float32 or not wc.is_contiguous():
        wc = wc.float().contiguous()
    call("b200seg_pack_weight", wc.data_ptr(), Cout, Cin, taps, out.data_ptr(), _dt(out),
         1 if transpose_flip else 0, co_off, co_total, layout, _stream())
    return out


def conv3d_fwd(x, x_coff, Cin, x_stats, act, wp, Cout, ksize, bias=None, residual=None, r_coff=0,
               want_stats=True, dgrad_of=None, algo=None, eps=IN_EPS):
    """y = conv(act(IN(x[..., x_coff:x_coff+Cin]))) (+bias)(+residual); returns (y, y_stats).
    wp: packed weights, either a tensor (DIRECT layout) or a (tensor, algo) pair from PackedWeights.
    dgrad_of=(tensor, coff, stats, act): data-gradient mode, see b200seg_conv3d_fwd."""
    _need_cuda(x)
    if isinstance(wp, tuple):
        wp, walgo = wp
        algo = walgo if algo is None else algo
    if algo is None:
        algo = ALGO_DIRECT
    B, D, H, W, x_ld = x.shape
    y = torch.empty(B, D, H, W, Cout, dtype=x.dtype, device=x.device)
    y_stats = new_stats(B, Cout, x.device) if want_stats else None
    gx = gcoff = gstats = None
    gact = ACT_NONE
    gld = 0
    if dgrad_of is not None:
        gx, gcoff, gstats, gact = dgrad_of
        gld = gx.shape[-1]
    call("b200seg_conv3d_fwd", x.data_ptr(), x_ld, x_coff, _p(x_stats), eps, act,
         wp.data_ptr(), _p(bias), _p(residual), 0 if residual is None else residual.shape[-1], r_coff,
         y.data_ptr(), Cout, 0, _p(y_stats),
         _p(gx), gld, gcoff or 0, _p(gstats), eps, gact,
         B, D, H, W, Cin, Cout, ksize[0], ksize[1], ksize[2], _dt(x), algo, _stream())
    return y, y_stats


def conv3d_wgrad(x, x_coff, Cin, x_stats, act, dy, dy_coff, Cout, ksize, want_bias=False,
                 algo=ALGO_AUTO, eps=IN_EPS):
    B, D, H, W, x_ld = x.shape
    dw = torch.zeros(Cout, Cin, ksize[0], ksize[1], ksize[2], dtype=torch.float32, device=x.device)
    db = torch.zeros(Cout, dtype=torch.float32, device=x.device) if want_bias else None
    normalised = 1 if (x_stats is not None or act) else 0
    ws_bytes = _lib.load().b200seg_conv3d_wgrad_workspace(x_ld, x_coff, normalised, dy.shape[-1], dy_coff,
                                                          1 if want_bias else 0, B, D, H, W, Cin, Cout,
                                                          ksize[0], ksize[1], ksize[2], _dt(x), algo)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
    call("b200seg_conv3d_wgrad", x.data_ptr(), x_ld, x_coff, _p(x_stats), eps, act,
         dy.data_ptr(), dy.shape[-1], dy_coff, dw.data_ptr(), _p(db),
         B, D, H, W, Cin, Cout, ksize[0], ksize[1], ksize[2], _dt(x), algo, _p(ws), ws_bytes, _stream())
    return dw, db


def in_bwd_apply(g, x, x_coff, C, x_stats, bstats, add=None, add_coff=0, out=None, out_coff=0, eps=IN_EPS):
    """dx = rstd*(g - S1/n - xhat*S2/n) (+ add); g is [B,D,H,W,C] dense."""
    B, D, H, W, _ = x.shape
    V = D * H * W
    if out is None:
        out = torch.empty(B, D, H, W, C, dtype=x.dtype, device=x.device)
    call("b200seg_instnorm_bwd_apply", g.data_ptr(), g.shape[-1], 0, x.data_ptr(), x.shape[-1], x_coff, _dt(x),
         x_stats.data_ptr(), bstats.data_ptr(), eps,
         _p(add), 0 if add is None else add.shape[-1], add_coff,
         out.data_ptr(), out.shape[-1], out_coff, B, V, C, _stream())
    return out


def in_apply(x, C, stats, act, eps=IN_EPS):
    """y = act(IN(x)) materialised (SingleConv post-activation)."""
    B, D, H, W, _ = x.shape
    y = torch.empty(B, D, H, W, C, dtype=x.dtype, device=x.device)
    call("b200seg_instnorm_apply", x.data_ptr(), _dt(x), x.shape[-1], 0, stats.data_ptr(), eps, act,
         y.data_ptr(), C, 0, B, D * H * W, C, _stream())
    return y


def in_bwd_reduce(dy, x, C, stats, act, eps=IN_EPS):
    """g = dy * act'(xhat) and the two IN-backward sums; returns (g, bstats)."""
    B, D, H, W, _ = x.shape
    g = torch.empty(B, D, H, W, C, dtype=x.dtype, device=x.device)
    bst = new_stats(B, C, x.device)
    call("b200seg_instnorm_bwd_reduce", dy.data_ptr(), dy.shape[-1], 0, x.data_ptr(), x.shape[-1], 0, _dt(x),
         stats.data_ptr(), eps, act, g.data_ptr(), C, 0, bst.data_ptr(), B, D * H * W, C, _stream())
    return g, bst


def copy_channels(x, x_coff, y, y_coff, C, accumulate=False):
    nvox = x.numel() // x.shape[-1]
    call("b200seg_copy_channels", x.data_ptr(), _dt(x), x.shape[-1], x_coff, y.data_ptr(), _dt(y), y.shape[-1],
         y_coff, 1 if accumulate else 0, nvox, C, _stream())
    return y


def instnorm_stats(x, x_coff, C):
    B, D, H, W, ld = x.shape
    st = new_stats(B, C, x.device)
    call("b200seg_instnorm_stats", x.data_ptr(), _dt(x), ld, x_coff, B, D * H * W, C, st.data_ptr(), _stream())
    return st


# ----------------------------------------------------------------------------- weight cache
class PackedWeights:
    """Per-module holder of the packed (fwd and dgrad) images of one (possibly fused) conv weight.

    Staleness rule (ADVICE r1, high): an in-place write through ``.data`` — the reference's own
    ``update_ema_variables`` (training/utils.py:99-102) — does not bump ``Tensor._version``, so version counters
    cannot prove an image fresh.  Instead the images are simply rebuilt on EVERY forward:
      * a holder attached to a ``PackRegistry`` (every b200seg model attaches its holders) is refreshed by the
        registry's single multi-tensor launch at the top of ``model.forward`` (≈60 us for 40 M parameters);
      * a free-standing holder (unit tests driving one block) re-packs inside ``get`` with per-weight launches.
    What IS cached is the allocation and the job description, keyed on (dtype, B, co_pad, the two algorithms,
    data_ptrs, shapes): the algorithms name the image layouts, so toggling TF32 repacks instead of handing one kernel
    the other's image."""

    def __init__(self):
        self._sig = None
        self._fwd = None
        self._bwd = None
        self._jobs = []           # [(weight, out tensor, transpose_flip, co_off, co_total, layout)]
        self._registry = None
        self._epoch = -1
        self._algo_key = None     # (dtype, B, co_pad, shapes, TF32 allowed) the cached algorithms were chosen for
        self._algo_pair = None

    def _algos(self, weights, dtype, B, co_pad):
        """(forward, data-gradient) algorithms, asked of the library only when an input of the choice changed"""
        key = (dtype, B, co_pad, tuple(tuple(w.shape) for w in weights), dtype != torch.float16 and tf32_enabled())
        if key != self._algo_key:
            co_total = sum(w.shape[0] for w in weights) + co_pad
            Cin, ks = weights[0].shape[1], tuple(weights[0].shape[2:])
            self._algo_key = key
            self._algo_pair = (conv_algo(Cin, co_total, ks, dtype, B),
                               conv_algo(co_total, Cin, ks, dtype, B))      # dgrad: channels swap roles
        return self._algo_pair

    def _signature(self, weights, dtype, B, co_pad, algos):
        return (dtype, B, co_pad, algos) + tuple((w.data_ptr(), tuple(w.shape)) for w in weights)

    def get(self, weights, dtype, B=1, co_pad=0):
        """co_pad extra all-zero output channels are appended (Cout not a multiple of 8/16, e.g. the 27 map codes
        or 14 classes of MedFormer) so the wide-tile kernels and 16-byte stores apply; callers ignore them."""
        algos = self._algos(weights, dtype, B, co_pad)
        sig = self._signature(weights, dtype, B, co_pad, algos)
        reg = self._registry
        if sig == self._sig and reg is not None and self._epoch == reg.epoch:
            return self._fwd, self._bwd           # refreshed by the registry's launch of this forward
        if sig != self._sig:
            co_total = sum(w.shape[0] for w in weights) + co_pad
            Cin = weights[0].shape[1]
            taps = weights[0][0, 0].numel()
            dev = weights[0].device
            algo_f, algo_b = algos
            alloc = torch.zeros if co_pad else torch.empty
            fwd = alloc(taps * co_total * Cin, dtype=dtype, device=dev)
            bwd = alloc(taps * co_total * Cin, dtype=dtype, device=dev)
            jobs, off = [], 0
            for w in weights:
                jobs.append((w, fwd, False, off, co_total, algo_f))
                jobs.append((w, bwd, True, off, co_total, algo_b))
                off += w.shape[0]
            self._sig, self._fwd, self._bwd, self._jobs = sig, (fwd, algo_f), (bwd, algo_b), jobs
            if reg is not None:
                reg.dirty = True
        for w, out, flip, off, co_total, layout in self._jobs:
            pack_weight(w, out.dtype, flip, out, off, co_total, layout)
        if reg is not None:
            self._epoch = reg.epoch
        return self._fwd, self._bwd


class PackRegistry:
    """All PackedWeights holders of one model; ``refresh()`` re-packs every known weight with one launch."""

    def __init__(self, model):
        self.holders = []
        for m in model.modules():
            for v in vars(m).values():
                for h in (v if isinstance(v, (list, tuple)) else (v,)):
                    if isinstance(h, PackedWeights) and h._registry is None:
                        h._registry = self
                        self.holders.append(h)
        self.epoch = 0
        self.dirty = True
        self._tables = None
        self._table_sig = None

    def refresh(self):
        """Start a new forward: every holder that already knows its jobs is refreshed here in one launch; holders
        seen for the first time (or whose dtype/batch changed) fall back to per-weight launches inside get()."""
        self.epoch += 1
        live = [h for h in self.holders if h._jobs]
        if not live or live[0]._jobs[0][0].device.type != "cuda":
            return                      # nothing known yet (first forward): get() packs lazily
        tsig = tuple(h._sig for h in live)
        if self.dirty or tsig != self._table_sig:
            lib = _lib.load()
            chunk = lib.b200seg_pack_chunk_elems()
            jobs, chunks = [], []
            for h in live:
                for w, out, flip, off, co_total, layout in h._jobs:
                    if w.dtype != torch.float32 or not w.is_contiguous():
                        raise _lib.B200SegError("conv weights must be contiguous fp32 parameters")
                    taps = w[0, 0].numel()
                    j = len(jobs)
                    jobs.append([w.data_ptr(), out.data_ptr(), w.shape[0], w.shape[1], taps, _dt(out),
                                 1 if flip else 0, off, co_total, _LAYOUT_CODE[layout]])
                    tile_ci = lib.b200seg_pack_tile_ci(taps)
                    if tile_ci and w.shape[0] % 8 == 0 and w.shape[1] % 8 == 0 and off % 8 == 0 and w.shape[1] < 65536:
                        # TILE chunks: 8 output channels x tile_ci input channels x all taps per block (16-byte stores)
                        chunks.extend([j, -(1 + co0 * 65536 + ci0)] for co0 in range(0, w.shape[0], 8)
                                      for ci0 in range(0, w.shape[1], tile_ci))
                    else:
                        chunks.extend([j, e] for e in range(0, w.numel(), chunk))
            dev = live[0]._jobs[0][0].device
            self._tables = (torch.tensor(jobs, dtype=torch.int64).to(dev), torch.tensor(chunks, dtype=torch.int64).to(dev),
                            len(chunks))
            self._table_sig, self.dirty = tsig, False
        jt, ct, n = self._tables
        with torch.cuda.device(jt.device):
            call("b200seg_pack_weights_multi", jt.data_ptr(), ct.data_ptr(), n, _stream())
        for h in live:
            h._epoch = self.epoch


# ----------------------------------------------------------------------------- autograd Functions
class StemConvFn(torch.autograd.Function):
    """Raw conv (no norm/act on the input) + IN sums of the output: `inconv.conv1`, unet_utils.py:14,18."""

    @staticmethod
    def forward(ctx, x, w, wp_fwd, ksize):
        Cout, Cin = w.shape[0], w.shape[1]
        y, st = conv3d_fwd(x, 0, Cin, None, ACT_NONE, wp_fwd, Cout, ksize)
        ctx.save_for_backward(x)
        ctx.meta = (Cin, Cout, ksize, x.requires_grad)
        ctx.mark_non_differentiable(st)
        return y, st

    @staticmethod
    def backward(ctx, dy, _):
        (x,) = ctx.saved_tensors
        Cin, Cout, ksize, _xg = ctx.meta
        dy = dy.contiguous()
        dw, _ = conv3d_wgrad(x, 0, Cin, None, ACT_NONE, dy, 0, Cout, ksize)
        # the network input needs no gradient (SURVEY.md §8d: "minus dgrad of the stem")
        return None, dw, None, None


class BasicBlockFn(torch.autograd.Function):
    """Pre-activation residual block, conv_layers.py:71-94:
         out = conv2(relu(IN(conv1(relu(IN(x)))))) + shortcut(x)
       shortcut = identity, or conv(relu(IN(x))) sharing conv1's normalised input -> one fused GEMM of
       width 2*Cout (conv_layers.py:79,84).  Forward = 2 conv launches; IN normalise+ReLU live in the
       conv loaders, residual add and the next layer's IN sums in the conv epilogues."""

    @staticmethod
    def forward(ctx, x, x_stats, w1, w2, wsc, packs, ksize, x_coff, Cin):
        Cout = w1.shape[0]
        has_sc = wsc is not None
        (wf_fwd, wf_bwd), (w2_fwd, w2_bwd) = packs
        Cf = 2 * Cout if has_sc else Cout
        ts, ts_stats = conv3d_fwd(x, x_coff, Cin, x_stats, ACT_RELU, wf_fwd, Cf, ksize)
        t1_stats = ts_stats[:, :Cout].contiguous() if has_sc else ts_stats
        if has_sc:
            out, out_stats = conv3d_fwd(ts, 0, Cout, t1_stats, ACT_RELU, w2_fwd, Cout, ksize, residual=ts, r_coff=Cout)
        else:
            out, out_stats = conv3d_fwd(ts, 0, Cout, t1_stats, ACT_RELU, w2_fwd, Cout, ksize, residual=x, r_coff=x_coff)
        ctx.save_for_backward(x, x_stats, ts, t1_stats, wf_bwd[0], w2_bwd[0])
        ctx.meta = (Cin, Cout, ksize, x_coff, has_sc, wf_bwd[1], w2_bwd[1])
        ctx.mark_non_differentiable(out_stats)
        return out, out_stats

    @staticmethod
    def backward(ctx, d_out, _):
        x, x_stats, ts, t1_stats, wf_bwd, w2_bwd = ctx.saved_tensors
        Cin, Cout, ksize, x_coff, has_sc, algo_f, algo_2 = ctx.meta
        wf_bwd, w2_bwd = (wf_bwd, algo_f), (w2_bwd, algo_2)
        d_out = d_out.contiguous()
        B, D, H, W, _ = d_out.shape
        # ---- conv2: out = conv(relu(IN(t1))) + shortcut
        dw2, _ = conv3d_wgrad(ts, 0, Cout, t1_stats, ACT_RELU, d_out, 0, Cout, ksize)
        g2, b2 = conv3d_fwd(d_out, 0, Cout, None, ACT_NONE, w2_bwd, Cout, ksize,
                            dgrad_of=(ts, 0, t1_stats, ACT_RELU))
        if has_sc:
            d_ts = torch.empty(B, D, H, W, 2 * Cout, dtype=d_out.dtype, device=d_out.device)
            in_bwd_apply(g2, ts, 0, Cout, t1_stats, b2, out=d_ts, out_coff=0)
            copy_channels(d_out, 0, d_ts, Cout, Cout)
            Cf = 2 * Cout
        else:
            d_ts = in_bwd_apply(g2, ts, 0, Cout, t1_stats, b2)
            Cf = Cout
        del g2
        # ---- fused conv1 (+shortcut): ts = conv(relu(IN(x)))
        dwf, _ = conv3d_wgrad(x, x_coff, Cin, x_stats, ACT_RELU, d_ts, 0, Cf, ksize)
        g1, b1 = conv3d_fwd(d_ts, 0, Cf, None, ACT_NONE, wf_bwd, Cin, ksize,
                            dgrad_of=(x, x_coff, x_stats, ACT_RELU))
        if has_sc:
            dx = in_bwd_apply(g1, x, x_coff, Cin, x_stats, b1)
            dw1, dwsc = dwf[:Cout], dwf[Cout:]
        else:
            dx = in_bwd_apply(g1, x, x_coff, Cin, x_stats, b1, add=d_out, add_coff=0)
            dw1, dwsc = dwf, None
        if x.shape[-1] != Cin:
            # x was a channel slice of a wider tensor: scatter the gradient back into that frame
            full = torch.zeros_like(x)
            copy_channels(dx, 0, full, x_coff, Cin)
            dx = full
        return dx, None, dw1, dw2, dwsc, None, None, None, None


class SingleConvFn(torch.autograd.Function):
    """SingleConv (post-activation), conv_layers.py:46-53,56-68: y = relu(IN(conv(x))).  The raw conv output
    and its IN sums are kept; the normalise+ReLU is materialised by one elementwise kernel."""

    @staticmethod
    def forward(ctx, x, w, packs, ksize, x_coff, Cin):
        Cout = w.shape[0]
        w_fwd, w_bwd = packs
        r, r_stats = conv3d_fwd(x, x_coff, Cin, None, ACT_NONE, w_fwd, Cout, ksize)
        y = in_apply(r, Cout, r_stats, ACT_RELU)
        ctx.save_for_backward(x, r, r_stats, w_bwd[0])
        ctx.meta = (Cin, Cout, ksize, x_coff, x.requires_grad, w_bwd[1])
        return y

    @staticmethod
    def backward(ctx, dy):
        x, r, r_stats, w_bwd = ctx.saved_tensors
        Cin, Cout, ksize, x_coff, need_dx, algo_b = ctx.meta
        w_bwd = (w_bwd, algo_b)
        dy = dy.contiguous()
        g, bst = in_bwd_reduce(dy, r, Cout, r_stats, ACT_RELU)
        dr = in_bwd_apply(g, r, 0, Cout, r_stats, bst)
        dw, _ = conv3d_wgrad(x, x_coff, Cin, None, ACT_NONE, dr, 0, Cout, ksize)
        dx = None
        if need_dx:
            dx, _ = conv3d_fwd(dr, 0, Cout, None, ACT_NONE, w_bwd, Cin, ksize, want_stats=False)
            if x.shape[-1] != Cin:
                full = torch.zeros_like(x)
                copy_channels(dx, 0, full, x_coff, Cin)
                dx = full
        return dx, dw, None, None, None, None


class MaxPoolFn(torch.autograd.Function):
    """nn.MaxPool3d(scale) (kernel == stride), unet_utils.py:36, + IN sums of the pooled tensor."""

    @staticmethod
    def forward(ctx, x, scale, want_stats):
        _need_cuda(x)
        B, D, H, W, C = x.shape
        sd, sh, sw = scale
        Do, Ho, Wo = D // sd, H // sh, W // sw
        y = torch.empty(B, Do, Ho, Wo, C, dtype=x.dtype, device=x.device)
        idx = torch.empty(B, Do, Ho, Wo, C, dtype=torch.uint8, device=x.device)
        st = new_stats(B, C, x.device) if want_stats else None
        call("b200seg_maxpool3d_fwd", x.data_ptr(), C, 0, y.data_ptr(), C, 0, idx.data_ptr(), _p(st),
             B, D, H, W, C, sd, sh, sw, _dt(x), _stream())
        ctx.save_for_backward(idx)
        ctx.meta = (B, D, H, W, C, scale)
        if st is None:
            st = torch.empty(0, device=x.device)
        ctx.mark_non_differentiable(st)
        return y, st

    @staticmethod
    def backward(ctx, dy, _):
        (idx,) = ctx.saved_tensors
        B, D, H, W, C, (sd, sh, sw) = ctx.meta
        dy = dy.contiguous()
        exact = (D % sd == 0) and (H % sh == 0) and (W % sw == 0)
        dx = (torch.empty if exact else torch.zeros)(B, D, H, W, C, dtype=dy.dtype, device=dy.device)
        call("b200seg_maxpool3d_bwd", dy.data_ptr(), C, 0, idx.data_ptr(), dx.data_ptr(), C, 0,
             B, D, H, W, C, sd, sh, sw, _dt(dy), _stream())
        return dx, None, None


class UpCatFn(torch.autograd.Function):
    """F.interpolate(x1, size=x2.shape, 'trilinear', align_corners=True) + cat([x2, x1]) (unet_utils.py:69-71)
    written straight into one concat buffer, with the IN sums of the upsampled channels."""

    @staticmethod
    def forward(ctx, low, skip, skip_stats, skip_first):
        _need_cuda(low)
        B, Di, Hi, Wi, Cl = low.shape
        _, Do, Ho, Wo, Cs = skip.shape
        cat = torch.empty(B, Do, Ho, Wo, Cs + Cl, dtype=low.dtype, device=low.device)
        s_off, u_off = (0, Cs) if skip_first else (Cl, 0)
        copy_channels(skip, 0, cat, s_off, Cs)
        up_stats = new_stats(B, Cl, low.device)
        call("b200seg_upsample_trilinear_fwd", low.data_ptr(), Cl, 0, cat.data_ptr(), Cs + Cl, u_off,
             up_stats.data_ptr(), B, Di, Hi, Wi, Do, Ho, Wo, Cl, _dt(low), _stream())
        if skip_stats is None or skip_stats.numel() == 0:
            skip_stats = instnorm_stats(skip, 0, Cs)
        cat_stats = torch.cat([skip_stats, up_stats] if skip_first else [up_stats, skip_stats], dim=1).contiguous()
        ctx.meta = (low.shape, skip.shape, s_off, u_off)
        ctx.mark_non_differentiable(cat_stats)
        return cat, cat_stats

    @staticmethod
    def backward(ctx, d_cat, _):
        (B, Di, Hi, Wi, Cl), (_, Do, Ho, Wo, Cs), s_off, u_off = ctx.meta
        d_cat = d_cat.contiguous()
        d_skip = torch.empty(B, Do, Ho, Wo, Cs, dtype=d_cat.dtype, device=d_cat.device)
        copy_channels(d_cat, s_off, d_skip, 0, Cs)
        d_low = torch.empty(B, Di, Hi, Wi, Cl, dtype=d_cat.dtype, device=d_cat.device)
        call("b200seg_upsample_trilinear_bwd", d_cat.data_ptr(), Cs + Cl, u_off, d_low.data_ptr(), Cl, 0, 0,
             B, Di, Hi, Wi, Do, Ho, Wo, Cl, _dt(d_cat), _stream())
        return d_low, d_skip, None, None


class OutConvFn(torch.autograd.Function):
    """1x1x1 conv with bias on the raw block output: `outc`, unet.py:47,62."""

    @staticmethod
    def forward(ctx, x, w, bias, packs):
        w_fwd, w_bwd = packs
        Cout, Cin = w.shape[0], w.shape[1]
        y, _ = conv3d_fwd(x, 0, Cin, None, ACT_NONE, w_fwd, Cout, (1, 1, 1), bias=bias, want_stats=False)
        ctx.save_for_backward(x, w_bwd[0])
        ctx.meta = (Cin, Cout, w_bwd[1])
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w_bwd = ctx.saved_tensors
        Cin, Cout, algo_b = ctx.meta
        w_bwd = (w_bwd, algo_b)
        dy = dy.contiguous()
        dw, db = conv3d_wgrad(x, 0, Cin, None, ACT_NONE, dy, 0, Cout, (1, 1, 1), want_bias=True)
        dx, _ = conv3d_fwd(dy, 0, Cout, None, ACT_NONE, w_bwd, Cin, (1, 1, 1), want_stats=False)
        return dx, dw, db, None


class DiceCEFn(torch.autograd.Function):
    """ce_scale*CrossEntropy(weight) + dice_scale*DiceLoss in one pass each way
    (training/losses.py:18-58, train_ddp.py:93,186-191)."""

    last_stats = None     # the kernel's stats buffer of the most recent forward ({loss, ce, dice, wsum}, dTP, dSP, alpha_c, dice_c)

    @staticmethod
    def forward(ctx, logits, labels, weight, ce_scale, dice_scale):
        _need_cuda(logits)
        if logits.dtype not in (torch.float16, torch.float32):
            logits = logits.float()
        B, C = logits.shape[0], logits.shape[1]
        V = logits[0, 0].numel()
        # accept both NCDHW-contiguous and channels-last (our model's output view) without copying
        lg = logits
        flat = lg.reshape(B, C, V) if lg.is_contiguous() else None
        if flat is not None:
            sb, sc, sv = C * V, V, 1
        else:
            perm = lg.permute(0, *range(2, lg.dim()), 1)
            if not perm.is_contiguous():
                lg = lg.contiguous()
                sb, sc, sv = C * V, V, 1
            else:
                sb, sc, sv = C * V, 1, C
        if labels.dtype == torch.int64:
            lb = 8
        elif labels.dtype == torch.uint8:
            lb = 1
        else:
            labels = labels.long()
            lb = 8
        labels = labels.contiguous()
        if labels.numel() != B * V:
            raise ValueError("labels must have B*V elements")
        dev = logits.device
        partial = torch.empty(3 * C + 2, dtype=torch.float64, device=dev)
        out = torch.empty(4 + 4 * C, dtype=torch.float32, device=dev)
        wt = None if weight is None else weight.to(device=dev, dtype=torch.float32).contiguous()
        call("b200seg_dice_ce_fwd", lg.data_ptr(), _dt(lg), sb, sv, sc, labels.data_ptr(), lb, _p(wt),
             B, V, C, float(ce_scale), float(dice_scale), partial.data_ptr(), out.data_ptr(), _stream())
        ctx.save_for_backward(lg, labels, out, wt if wt is not None else torch.empty(0, device=dev))
        ctx.meta = (B, V, C, sb, sv, sc, lb, float(ce_scale), float(dice_scale), wt is not None, logits.shape)
        DiceCEFn.last_stats = out
        return out[0].clone()

    @staticmethod
    def backward(ctx, g):
        lg, labels, out, wt = ctx.saved_tensors
        B, V, C, sb, sv, sc, lb, ce_scale, dice_scale, has_w, shape = ctx.meta
        d = torch.empty_like(lg)  # preserves strides (channels-last or contiguous)
        gg = g.detach().to(torch.float32).contiguous()
        call("b200seg_dice_ce_bwd", lg.data_ptr(), _dt(lg), sb, sv, sc, labels.data_ptr(), lb,
             wt.data_ptr() if has_w else None, B, V, C, ce_scale, dice_scale, out.data_ptr(), gg.data_ptr(),
             d.data_ptr(), _stream())
        return d.view(shape) if d.shape != shape else d, None, None, None, None


# ----------------------------------------------------------------------------- MedFormer B-MHA core
def biattn_fwd(fqv, mqv, heads, dim_head=32):
    """fqv [B,D,H,W,2*inner], mqv [B,md,mh,mw,2*inner] channels-last (q block first, then v — the chunk(2, dim=1)
    of medformer_utils.py:67-68).  Returns feat_out [B,D,H,W,inner], map_out [B,md,mh,mw,inner], colstat."""
    _need_cuda(fqv)
    inner = heads * dim_head
    B = fqv.shape[0]
    N = fqv.numel() // (B * fqv.shape[-1])
    M = mqv.numel() // (B * mqv.shape[-1])
    assert fqv.shape[-1] == 2 * inner and mqv.shape[-1] == 2 * inner and fqv.dtype == mqv.dtype
    fo = torch.empty(*fqv.shape[:-1], inner, dtype=fqv.dtype, device=fqv.device)
    mo = torch.empty(*mqv.shape[:-1], inner, dtype=fqv.dtype, device=fqv.device)
    colstat = torch.empty(B, heads, M, 2, dtype=torch.float32, device=fqv.device)
    ws = torch.empty(_lib.load().b200seg_biattn_workspace(B, N, M, heads), dtype=torch.uint8, device=fqv.device)
    call("b200seg_biattn_fwd", fqv.data_ptr(), 2 * inner, 0, fqv.data_ptr(), 2 * inner, inner,
         mqv.data_ptr(), 0, mqv.data_ptr(), inner, 2 * inner, fo.data_ptr(), inner, 0, mo.data_ptr(), inner, 0,
         colstat.data_ptr(), ws.data_ptr(), B, N, M, heads, dim_head, float(dim_head) ** -0.5, _dt(fqv), _stream())
    return fo, mo, colstat


def biattn_bwd(fqv, mqv, mo, colstat, dfo, dmo, heads, dim_head=32):
    inner = heads * dim_head
    B = fqv.shape[0]
    N = fqv.numel() // (B * fqv.shape[-1])
    M = mqv.numel() // (B * mqv.shape[-1])
    dfqv = torch.empty_like(fqv)
    dmqv = torch.empty_like(mqv)
    ws = torch.empty(_lib.load().b200seg_biattn_workspace(B, N, M, heads), dtype=torch.uint8, device=fqv.device)
    call("b200seg_biattn_bwd", fqv.data_ptr(), 2 * inner, 0, fqv.data_ptr(), 2 * inner, inner,
         mqv.data_ptr(), 0, mqv.data_ptr(), inner, 2 * inner, mo.data_ptr(), inner, 0, colstat.data_ptr(),
         dfo.data_ptr(), inner, 0, dmo.data_ptr(), inner, 0,
         dfqv.data_ptr(), 2 * inner, 0, dfqv.data_ptr(), 2 * inner, inner,
         dmqv.data_ptr(), 0, dmqv.data_ptr(), inner, 2 * inner,
         ws.data_ptr(), B, N, M, heads, dim_head, float(dim_head) ** -0.5, _dt(fqv), _stream())
    return dfqv, dmqv


def biattn_wide_fwd(fqv, mqv, heads, dim_head):
    """biattn_fwd for the shapes b200seg_biattn_fwd refuses (dim_head 64 / 80, or more than 64 map tokens at 32)."""
    _need_cuda(fqv)
    inner = heads * dim_head
    B = fqv.shape[0]
    N = fqv.numel() // (B * fqv.shape[-1])
    M = mqv.numel() // (B * mqv.shape[-1])
    assert fqv.shape[-1] == 2 * inner and mqv.shape[-1] == 2 * inner and fqv.dtype == mqv.dtype
    fo = torch.empty(*fqv.shape[:-1], inner, dtype=fqv.dtype, device=fqv.device)
    mo = torch.empty(*mqv.shape[:-1], inner, dtype=fqv.dtype, device=fqv.device)
    colstat = torch.empty(B, heads, M, 2, dtype=torch.float32, device=fqv.device)
    ws = torch.empty(_lib.load().b200seg_biattn_wide_workspace(B, N, M, heads, dim_head), dtype=torch.uint8,
                     device=fqv.device)
    call("b200seg_biattn_wide_fwd", fqv.data_ptr(), 2 * inner, 0, fqv.data_ptr(), 2 * inner, inner,
         mqv.data_ptr(), 0, mqv.data_ptr(), inner, 2 * inner, fo.data_ptr(), inner, 0, mo.data_ptr(), inner, 0,
         colstat.data_ptr(), ws.data_ptr(), B, N, M, heads, dim_head, float(dim_head) ** -0.5, _dt(fqv), _stream())
    return fo, mo, colstat


def biattn_wide_bwd(fqv, mqv, mo, colstat, dfo, dmo, heads, dim_head):
    inner = heads * dim_head
    B = fqv.shape[0]
    N = fqv.numel() // (B * fqv.shape[-1])
    M = mqv.numel() // (B * mqv.shape[-1])
    dfqv = torch.empty_like(fqv)
    dmqv = torch.empty_like(mqv)
    ws = torch.empty(_lib.load().b200seg_biattn_wide_workspace(B, N, M, heads, dim_head), dtype=torch.uint8,
                     device=fqv.device)
    call("b200seg_biattn_wide_bwd", fqv.data_ptr(), 2 * inner, 0, fqv.data_ptr(), 2 * inner, inner,
         mqv.data_ptr(), 0, mqv.data_ptr(), inner, 2 * inner, mo.data_ptr(), inner, 0, colstat.data_ptr(),
         dfo.data_ptr(), inner, 0, dmo.data_ptr(), inner, 0,
         dfqv.data_ptr(), 2 * inner, 0, dfqv.data_ptr(), 2 * inner, inner,
         dmqv.data_ptr(), 0, dmqv.data_ptr(), inner, 2 * inner,
         ws.data_ptr(), B, N, M, heads, dim_head, float(dim_head) ** -0.5, _dt(fqv), _stream())
    return dfqv, dmqv


def biattn_is_wide(dim_head, M):
    """Which B-MHA entry owns a shape: the original one-voxel-per-thread kernels keep dim_head 32 with <= 64 map tokens
    (every BCV / AMOS / KiTS level, bit for bit as before); everything else goes to the wide kernels."""
    return not (dim_head == 32 and M <= 64)


class BiAttnFn(torch.autograd.Function):
    """Differentiable B-MHA core on channels-last tensors (medformer_utils.py:63-97 minus the projections)."""

    @staticmethod
    def forward(ctx, fqv, mqv, heads, dim_head):
        fqv = fqv.contiguous()
        mqv = mqv.contiguous()
        wide = biattn_is_wide(dim_head, mqv.numel() // (mqv.shape[0] * mqv.shape[-1]))
        fo, mo, colstat = (biattn_wide_fwd if wide else biattn_fwd)(fqv, mqv, heads, dim_head)
        ctx.save_for_backward(fqv, mqv, mo, colstat)
        ctx.hd = (heads, dim_head)
        ctx.wide = wide
        return fo, mo

    @staticmethod
    def backward(ctx, dfo, dmo):
        fqv, mqv, mo, colstat = ctx.saved_tensors
        bwd = biattn_wide_bwd if ctx.wide else biattn_bwd
        dfqv, dmqv = bwd(fqv, mqv, mo, colstat, dfo.contiguous(), dmo.contiguous(), *ctx.hd)
        return dfqv, dmqv, None, None


# ----------------------------------------------------------------------------- depthwise conv (MedFormer)
def dwconv3d(x, w_taps, ksize, x_stats=None, act=ACT_NONE, flip=False, want_stats=False, eps=IN_EPS, cmajor=False):
    """x [B,D,H,W,C] channels-last; w_taps float32 [taps][C], or with cmajor the module's own [C,1,kd,kh,kw] parameter
    read in place (no transposed copy per call).  Returns (y, y_stats or None)."""
    _need_cuda(x)
    B, D, H, W, C = x.shape
    y = torch.empty_like(x)
    st = new_stats(B, C, x.device) if want_stats else None
    call("b200seg_dwconv3d_fwd", x.data_ptr(), C, 0, _p(x_stats), eps, act, w_taps.data_ptr(), (1 if flip else 0) | (2 if cmajor else 0),
         y.data_ptr(), C, 0, _p(st), B, D, H, W, C, ksize[0], ksize[1], ksize[2], _dt(x), _stream())
    return y, st


def dwconv3d_wgrad(x, dy, ksize, x_stats=None, act=ACT_NONE, eps=IN_EPS, cmajor=False):
    """dw as [taps][C], or with cmajor as [C,1,kd,kh,kw] — directly the parameter's gradient."""
    B, D, H, W, C = x.shape
    taps = ksize[0] * ksize[1] * ksize[2]
    dw = torch.zeros((C, 1, *ksize) if cmajor else (taps, C), dtype=torch.float32, device=x.device)
    call("b200seg_dwconv3d_wgrad", x.data_ptr(), C, 0, _p(x_stats), eps, act, dy.data_ptr(), C, 0, dw.data_ptr(), 1 if cmajor else 0,
         B, D, H, W, C, ksize[0], ksize[1], ksize[2], _dt(x), _stream())
    return dw


def dw_weight(weight):
    """The depthwise parameter as the kernels take it: in place when it is a contiguous fp32 tensor (every module of the
    package), otherwise one fp32 copy.  Always [C,1,kd,kh,kw] (cmajor)."""
    w = weight.detach()
    if w.dtype != torch.float32 or not w.is_contiguous():
        w = w.float().contiguous()
    return w


class DepthwiseConvFn(torch.autograd.Function):
    """nn.Conv3d(C, C, k, padding=k//2, groups=C, bias=False) on a channels-last tensor (conv_layers.py:135-143).
    weight is the module's own [C,1,kd,kh,kw] parameter, so state_dicts stay interchangeable."""

    @staticmethod
    def forward(ctx, x, weight):
        ks = tuple(weight.shape[2:])
        wt = dw_weight(weight)
        x = x.contiguous()
        y, _ = dwconv3d(x, wt, ks, cmajor=True)
        ctx.save_for_backward(x, wt)
        ctx.ks = ks
        ctx.wdtype = weight.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wt = ctx.saved_tensors
        dy = dy.contiguous()
        dx, _ = dwconv3d(dy, wt, ctx.ks, flip=True, cmajor=True)
        dw = dwconv3d_wgrad(x, dy, ctx.ks, cmajor=True)
        return dx, dw.to(ctx.wdtype)
