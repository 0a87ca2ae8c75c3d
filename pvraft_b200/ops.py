"""Tensor-level wrappers over the C ABI (include/pvraft_b200.h).

PyTorch is plumbing here: it owns device memory and the CUDA stream; every arithmetic step of the
hot path happens inside libpvraft_b200.so.  All wrappers require contiguous CUDA tensors and raise
on anything else -- there is deliberately no CPU / eager fallback.
"""
import ctypes as C
import threading
import weakref
from typing import NamedTuple

import torch

from . import _lib
from ._lib import (ACT_LRELU, ACT_NONE, ACT_RELU, IN_GN, IN_GN_MINMAX, IN_PLAIN, KNN, MOMENTS, check, lib)

launch_count = 0   # C-ABI calls that launch a kernel (bench.py reports it as gpu_launches)


def _stream():
    """The current stream of the CURRENT device: the library launches on the current device, so every operand has to live
    there (`_p` checks it) -- RSF.forward enters `torch.cuda.device(input.device)` itself; callers of the inner modules on
    a non-default GPU do the same (or `torch.cuda.set_device`), as under DDP / DataParallel."""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t, dtype=torch.float32):
    if t is None:
        return None
    if not torch.is_tensor(t):
        raise TypeError(f'expected a tensor, got {type(t)}')
    if not t.is_cuda:
        raise _lib.PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')
    if t.device.index != torch.cuda.current_device():
        raise _lib.PvraftError(f'tensor on {t.device} but the current CUDA device is {torch.cuda.current_device()}: the kernels '
                               'launch on the current device -- wrap the call in `with torch.cuda.device(t.device):`')
    if t.dtype != dtype:
        raise TypeError(f'expected {dtype}, got {t.dtype}')
    if not t.is_contiguous():
        raise ValueError('expected a contiguous tensor')
    return t.data_ptr()


def _count(rc, what):
    global launch_count
    check(rc, what)
    launch_count += 1


def deterministic():
    """True while torch.use_deterministic_algorithms(True) is in effect.  The wrappers that reduce floating-point values
    then hand the library a det_workspace (include/pvraft_b200.h, "Deterministic mode"), which makes their results bitwise
    reproducible; read at every call, so the flag can change between calls."""
    return torch.are_deterministic_algorithms_enabled()


def _det_workspace(size_fn, *size_args, device):
    """The det_workspace argument of a reducing entry point: while deterministic() is on, a zero-filled buffer of
    size_fn(*size_args) bytes (size_fn: the entry point's pvraft_*_det_workspace_bytes query); None otherwise."""
    if not deterministic():
        return None
    return torch.zeros(int(size_fn(*size_args)), dtype=torch.uint8, device=device)


_TLS = threading.local()   # .arena = [buffer [n,B,8,2] f64, next free block]: zeroed accumulators handed out inside a
                           # `stats_arena` scope (per thread: nn.DataParallel runs one replica per thread)


class stats_arena:
    """Scope in which `new_stats` (and the lookup's moment accumulator) are slices of ONE zero-filled buffer instead of a
    memset launch each: the RAFT loop needs 5 blocks per iteration (`with ops.stats_arena(b, dev, 5 * iters)`)."""

    def __init__(self, b, device, blocks):
        self.buf = [torch.zeros(blocks, b, 8, 2, dtype=torch.float64, device=device), 0]

    def __enter__(self):
        self.prev = getattr(_TLS, 'arena', None)
        _TLS.arena = self.buf
        return self

    def __exit__(self, *exc):
        _TLS.arena = self.prev
        return False


class bf16_compute:
    """Scope in which tc_weights returns the bf16 operand form of a layer's weights by default, so that every tensor-core
    layer (tc_linear, update_chain) launched inside it runs on bf16 operands with fp32 accumulation.  The RAFT loop enters it
    in the 'bf16-compute' precision mode (RSF.set_precision); the encoders and the refiner run outside it.  Per thread, like
    stats_arena."""

    def __init__(self, enabled=True):
        self.enabled = bool(enabled)

    def __enter__(self):
        self.prev = getattr(_TLS, 'bf16', False)
        _TLS.bf16 = self.enabled
        return self

    def __exit__(self, *exc):
        _TLS.bf16 = self.prev
        return False


def bf16_compute_active():
    """True inside an enabled `bf16_compute` scope on this thread."""
    return bool(getattr(_TLS, 'bf16', False))


def new_stats(b, device, n=1):
    """Zeroed GroupNorm accumulators: n x [B,8,2] doubles (one cudaMemset for all of them)."""
    arena = getattr(_TLS, 'arena', None)
    if arena is not None:
        buf, pos = arena
        if pos + n <= buf.shape[0] and buf.shape[1] == b and buf.device == torch.device(device):
            arena[1] = pos + n
            return buf[pos:pos + n]
    return torch.zeros(n, b, 8, 2, dtype=torch.float64, device=device)


def corr_reorder(val, idx):
    """Bank-aware permutation of every row of the truncated state (val [B,N,K] f32, idx [B,N,K] int32)."""
    b, n, k = val.shape
    val_out, idx_out = torch.empty_like(val), torch.empty_like(idx)
    _count(lib().pvraft_corr_reorder(_p(val), _p(idx, torch.int32), b * n, k, _p(val_out), _p(idx_out, torch.int32), _stream()),
           'corr_reorder')
    return val_out, idx_out


def corr_state_pack_bf16(val, idx, m=None):
    """Reordered fp32 / int32 state -> (bf16 values, uint16 ids held in an int16 tensor): 4 B per candidate and iteration.
    The ids are rows of the second cloud, so its size `m` (default: the rows of the state, i.e. clouds of equal size) is what
    the 16-bit ids must address."""
    m = int(idx.shape[1]) if m is None else int(m)
    if m > 65536:
        raise ValueError(f'uint16 candidate ids need a second cloud of at most 65536 points (N2 <= 65536), got {m}')
    v16 = torch.empty(val.shape, dtype=torch.bfloat16, device=val.device)
    i16 = torch.empty(idx.shape, dtype=torch.int16, device=idx.device)
    _count(lib().pvraft_corr_state_pack_bf16(_p(val), _p(idx, torch.int32), val.numel(), _p(v16, torch.bfloat16), _p(i16, torch.int16),
                                             _stream()), 'corr_state_pack_bf16')
    return v16, i16


def corr_matmul(fmap1_pm, fmap2_pm):
    """Point-major feature maps [B,N,C] x [B,M,C] -> all-pairs correlation [B,N,M] / sqrt(C) on wgmma (3xTF32)."""
    b, n, c = fmap1_pm.shape
    m = fmap2_pm.shape[1]
    if fmap2_pm.shape != (b, m, c):
        raise ValueError(f'corr_matmul: feature maps {tuple(fmap1_pm.shape)} and {tuple(fmap2_pm.shape)}')
    corr = torch.empty(b, n, m, dtype=torch.float32, device=fmap1_pm.device)
    ws = torch.empty(int(lib().pvraft_corr_matmul_workspace_bytes(b, n, m, c)), dtype=torch.uint8, device=fmap1_pm.device)
    _count(lib().pvraft_corr_matmul_fwd(_p(fmap1_pm), _p(fmap2_pm), b, n, m, c, _p(corr), _p(ws, torch.uint8), _stream()),
           'corr_matmul')
    return corr


def corr_topk(corr, k):
    """corr [B,N,M] -> (val [B,N,K] f32, idx [B,N,K] int32): the K largest per row, ascending column order."""
    b, n, m = corr.shape
    val = torch.empty(b, n, k, dtype=torch.float32, device=corr.device)
    idx = torch.empty(b, n, k, dtype=torch.int32, device=corr.device)
    _count(lib().pvraft_corr_topk_fwd(_p(corr), b, n, m, k, _p(val), _p(idx, torch.int32), _stream()), 'corr_topk')
    return val, idx


def corr_dense(fmap1_pm, fmap2_pm):
    """corr_matmul for any N and M: each ragged size is zero-padded on its own to the next multiple of 128 (the kernel's
    tile), and the result cropped."""
    n, m = fmap1_pm.shape[1], fmap2_pm.shape[1]
    pad_n, pad_m = (-n) % 128, (-m) % 128
    if pad_n == 0 and pad_m == 0:
        return corr_matmul(fmap1_pm, fmap2_pm)
    f1 = torch.nn.functional.pad(fmap1_pm, (0, 0, 0, pad_n)).contiguous()
    f2 = torch.nn.functional.pad(fmap2_pm, (0, 0, 0, pad_m)).contiguous()
    return corr_matmul(f1, f2)[:, :n, :m].contiguous()


CORR_ROW_MAX = 49152      # widest row the top-K kernels stage in shared memory (csrc/corr_topk.cu)
# Bytes of the windowed build's scratch: the correlation slab of one row block and window plus the row block's candidate
# lists.  A forward captured into a CUDA graph keeps this memory in its pool for as long as the graph lives, so the cap is a
# fixed, modest size rather than a share of the free memory; row blocks of >= 1800 rows keep every GEMM launch at more
# than ten 128 x 128 tiles per SM.
CORR_SLAB_CAP = 1 << 30


class CorrPlan(NamedTuple):
    """How corr_build computes the truncated correlation of a [B,N,C] x [B,M,C] pair.
    dense: one [B,N,M] matrix (corr_dense) and one corr_topk, as long as a whole row fits the top-K kernels (M <= 49152).
    Otherwise, for every sample and row block of fmap1, the slab of each column window of fmap2 is computed and reduced to its
    K best candidates, and the W*K candidates of a row are reduced to the row's K best: the same result as the dense build."""
    dense: bool
    windows: tuple      # ((c0, width), ...) column windows of fmap2, in ascending order, tiling [0, M); starts are 128-aligned
    row_blocks: tuple   # ((r0, rows), ...) row blocks of fmap1, in ascending order, tiling [0, N); starts are 128-aligned
    ld: int             # slab row stride in floats (the widest window; a multiple of 128)
    slab_bytes: int     # scratch: the [B,N,M] matrix (dense) or one row block's slab + candidate lists (windowed)


def _pad128(x):
    return (x + 127) // 128 * 128


def corr_plan(b, n, m, c, k, window=CORR_ROW_MAX, cap=CORR_SLAB_CAP):
    """Plan of corr_build for B samples of N x M correlations over C channels, truncated to K per row.  `window` (the widest
    column window, a multiple of 128) and `cap` (bytes of slab + candidate lists) exist for tests; the model uses the defaults."""
    if min(b, n, m, c, k) <= 0:
        raise ValueError(f'corr_plan: bad shape B={b} N={n} M={m} C={c} K={k}')
    if window % 128 or not 0 < window <= CORR_ROW_MAX:
        raise ValueError(f'corr_plan: window={window} must be a multiple of 128 and at most {CORR_ROW_MAX}')
    if m <= window:
        return CorrPlan(True, ((0, m),), ((0, n),), _pad128(m), 4 * b * _pad128(n) * _pad128(m))
    if k > m:
        raise ValueError(f'truncate_k={k} exceeds the number of points {m}')
    w = -(-m // window)
    if w * k > CORR_ROW_MAX:
        raise ValueError(f'a cloud of {m} points needs {w} column windows, and their {w * k} candidates per row exceed the '
                         f'{CORR_ROW_MAX} the merge step can stage (truncate_k={k}: at most {CORR_ROW_MAX // k * window} points)')
    width = _pad128(-(-m // w))   # <= window, and (w - 1) * width < m
    windows = tuple((i * width, min(width, m - i * width)) for i in range(w))
    if windows[-1][1] < k:
        raise ValueError(f'corr_plan: the last column window has {windows[-1][1]} columns, fewer than truncate_k={k}')
    per_row = 4 * width + 8 * w * k   # slab row + candidate values and ids
    rows = max(128, cap // per_row // 128 * 128)
    nb = -(-_pad128(n) // rows)
    rows = _pad128(-(-n // nb))
    row_blocks = tuple((r0, min(rows, n - r0)) for r0 in range(0, n, rows))
    return CorrPlan(False, windows, row_blocks, width, rows * per_row)


def corr_build(fmap1_pm, fmap2_pm, k, plan=None):
    """Point-major feature maps [B,N,C] x [B,M,C] -> (val [B,N,K] f32, idx [B,N,K] int32 rows of fmap2): the K largest
    correlations of every row, in ascending column order (corr_topk of corr_dense), without the [B,N,M] matrix when
    M > 49152 (see CorrPlan).  Both paths give the same bits."""
    b, n, c = fmap1_pm.shape
    m = fmap2_pm.shape[1]
    if fmap2_pm.dim() != 3 or fmap2_pm.shape[0] != b or fmap2_pm.shape[2] != c:
        raise ValueError(f'corr_build: feature maps {tuple(fmap1_pm.shape)} and {tuple(fmap2_pm.shape)} (same batch and channels)')
    if k > m:
        raise ValueError(f'truncate_k={k} exceeds the number of points {m} of the second cloud')
    if c % 32 != 0:
        raise NotImplementedError(f'calculate_corr: {c} feature channels (the wgmma GEMM needs a multiple of 32; the model has 128)')
    plan = corr_plan(b, n, m, c, k) if plan is None else plan
    if plan.dense:
        return corr_topk(corr_dense(fmap1_pm, fmap2_pm), k)
    dev = fmap1_pm.device
    npad, mpad = _pad128(n), _pad128(m)
    # tf32 hi/lo of both maps, split once, each map's rows per sample padded to 128 on their own.  The padding rows are left
    # unset: a row of A or B only reaches the slab entries of that row / column, and the top-K steps never read the entries
    # past N / M.
    ws_a = torch.empty(2, b, npad, c, dtype=torch.float32, device=dev)
    ws_b = torch.empty(2, b, mpad, c, dtype=torch.float32, device=dev)
    for ws, f, rows_f in ((ws_a, fmap1_pm, n), (ws_b, fmap2_pm, m)):
        for s in range(b):
            _count(lib().pvraft_tf32_split_fwd(_p(f[s]), rows_f * c, _p(ws[0, s]), _p(ws[1, s]), _stream()), 'tf32_split')
    nw = len(plan.windows)
    wk = nw * k
    rows = max(r for _, r in plan.row_blocks)
    slab = torch.empty(_pad128(rows), plan.ld, dtype=torch.float32, device=dev)
    cand_val = torch.empty(rows, wk, dtype=torch.float32, device=dev)
    cand_idx = torch.empty(rows, wk, dtype=torch.int32, device=dev)
    val = torch.empty(b, n, k, dtype=torch.float32, device=dev)
    idx = torch.empty(b, n, k, dtype=torch.int32, device=dev)
    for s in range(b):
        split = [_p(ws_a[0, s]), _p(ws_a[1, s]), _p(ws_b[0, s]), _p(ws_b[1, s])]
        for r0, nr in plan.row_blocks:
            for j, (c0, nc) in enumerate(plan.windows):
                _count(lib().pvraft_corr_matmul_window_fwd(*split, 1, npad, mpad, c, r0, nr, c0, nc, _p(slab), plan.ld, _stream()),
                       'corr_matmul_window')
                _count(lib().pvraft_corr_topk_window_fwd(_p(slab), nr, nc, plan.ld, k, c0, None, _p(cand_val) + 4 * j * k,
                                                         _p(cand_idx, torch.int32) + 4 * j * k, wk, _stream()), 'corr_topk_window')
            _count(lib().pvraft_corr_topk_window_fwd(_p(cand_val), nr, wk, wk, k, 0, _p(cand_idx, torch.int32), _p(val[s, r0:r0 + nr]),
                                                     _p(idx[s, r0:r0 + nr], torch.int32), k, _stream()), 'corr_topk_merge')
    return val, idx


def _table_rows(xyz2_pad, b):
    """M, the points of the second cloud, from its gather table [B,M,4]."""
    if xyz2_pad.dim() != 3 or xyz2_pad.shape[0] != b or xyz2_pad.shape[2] != 4:
        raise ValueError(f'expected a gather table [B={b},M,4], got {tuple(xyz2_pad.shape)}')
    return int(xyz2_pad.shape[1])


def check_pair(xyz1, xyz2, truncate_k):
    """The shape rules of a pair of clouds p = [xyz1 [B,N1,3], xyz2 [B,N2,3]]: one batch size, at least 32 points in each
    cloud (the 32-neighbour graphs) and at least truncate_k points in the second (the candidates of a row are distinct
    rows of xyz2).  N1 and N2 may differ; within a batch every sample has the same N1 and the same N2."""
    if xyz1.dim() != 3 or xyz1.shape[-1] != 3 or xyz2.dim() != 3 or xyz2.shape[-1] != 3:
        raise ValueError(f'expected p = [xyz1 [B,N1,3], xyz2 [B,N2,3]], got {tuple(xyz1.shape)} and {tuple(xyz2.shape)}')
    if xyz1.shape[0] != xyz2.shape[0]:
        raise ValueError(f'xyz1 {tuple(xyz1.shape)} and xyz2 {tuple(xyz2.shape)} must have the same batch size')
    n1, n2 = int(xyz1.shape[1]), int(xyz2.shape[1])
    if min(n1, n2) < KNN:
        raise ValueError(f'need at least {KNN} points per cloud, got N1={n1} and N2={n2}')
    if truncate_k > n2:
        raise ValueError(f'truncate_k={truncate_k} exceeds the number of points {n2} of the second cloud')


def xyz_pad(xyz):
    """[B,N,3] -> [B,N,4] = (x,y,z,0): the lookup kernel's gather table (one 128-bit load per candidate), built once per forward."""
    b, n, _ = xyz.shape
    out = torch.empty(b, n, 4, dtype=torch.float32, device=xyz.device)
    _count(lib().pvraft_xyz_pad_fwd(_p(xyz), b * n, _p(out), _stream()), 'xyz_pad')
    return out


def corr_lookup(corr_val, corr_idx, xyz2_pad, coords, levels, base_scale, vox=None, knn_sel=None, moments=None,
                want_slots=False, want_cube=False, vox_ld=None):
    """State [B,N,K], gather table xyz2_pad [B,M,4] of the second cloud, query coords [B,N,3]
    -> dict(vox [B,N,pad4(levels*27)], knn_sel [B,N,32,4], moments [B,16] f64, [knn_slot], [cube]).
    `cube` [B,N,K,levels] int8 is the fused kernel's own cell decision for every candidate (test hook)."""
    b, n, k = corr_val.shape
    m = _table_rows(xyz2_pad, b)
    dev = corr_val.device
    if vox_ld is None:
        vox_ld = (levels * 27 + 3) // 4 * 4      # rows padded to a multiple of 4 floats (zero-filled by the kernel)
    if vox is None:
        vox = torch.empty(b, n, vox_ld, dtype=torch.float32, device=dev)
    if knn_sel is None:
        knn_sel = torch.empty(b, n, KNN, 4, dtype=torch.float32, device=dev)
    if moments is None:
        moments = new_stats(b, dev, 1).view(b, MOMENTS) if MOMENTS == 16 else torch.zeros(b, MOMENTS, dtype=torch.float64, device=dev)
    slots = torch.empty(b, n, KNN, dtype=torch.int32, device=dev) if want_slots else None
    cube = torch.empty(b, n, k, levels, dtype=torch.int8, device=dev) if want_cube else None
    half = corr_val.dtype == torch.bfloat16   # reduced-precision state: bf16 values + uint16 ids (stored as int16)
    state = (_p(corr_val, torch.bfloat16), _p(corr_idx, torch.int16)) if half else (_p(corr_val), _p(corr_idx, torch.int32))
    fn = lib().pvraft_corr_lookup_bf16_fwd if half else lib().pvraft_corr_lookup_fwd
    ws = _det_workspace(lib().pvraft_corr_lookup_det_workspace_bytes, b, device=dev)
    _count(fn(*state, _p(xyz2_pad), _p(coords), b, n, m, k, levels, float(base_scale), _p(vox), vox.shape[-1], _p(knn_sel),
              _p(slots, torch.int32), _p(moments, torch.float64), _p(cube, torch.int8), _p(ws, torch.uint8), _stream()), 'corr_lookup')
    return dict(vox=vox, knn_sel=knn_sel, moments=moments, knn_slot=slots, cube=cube)


def linear(x, weight, bias=None, *, cin=None, w_ld=0, w_cin=0, in_mode=IN_PLAIN, in_min=None, in_stats=None, in_gamma=None,
           in_beta=None, in_count=0.0, in_act=ACT_NONE, in_slope=0.0, out_act=ACT_NONE, out=None, out_stats=None,
           residual=None, cout=None):
    """Fused [GN -> act ->] 1x1 conv [+bias] [-> ReLU] [+ residual] over x [B,N,cin] -> [B,N,cout]."""
    b, n, c = x.shape
    cin = c if cin is None else cin
    cout = weight.shape[0] if cout is None else cout
    if out is None:
        out = torch.empty(b, n, cout, dtype=torch.float32, device=x.device)
    a = _lib.LinearArgs(_p(x), _p(in_min), _p(in_stats, torch.float64), _p(in_gamma), _p(in_beta), float(in_count),
                        in_mode, in_act, float(in_slope), _p(weight), int(w_ld), int(w_cin), _p(bias), _p(residual), out_act,
                        _p(out), _p(out_stats, torch.float64), b, n, cin, cout)
    ws = _det_workspace(lib().pvraft_linear_det_workspace_bytes, b, device=x.device) if out_stats is not None else None
    _count(lib().pvraft_linear_fwd(C.byref(a), _p(ws, torch.uint8), _stream()), 'linear')
    return out


_TC_WEIGHTS = {}
TC_PLAIN, TC_GRU_ZR, TC_GRU_Q, TC_FLOW = 0, 1, 2, 3


def tc_weights(weights, col0=0, cols=None, k_pad=None, kcat=False, transposed=None, bf16=None):
    """tf32 hi/lo split of a (stack of) [cout, cin(,1,1)] weight(s) -> (hi, lo, n_pad, rows), hi and lo [n_pad, k_pad],
    cached per parameter version (inference weights are static, so this runs once; the training path re-splits after every
    optimizer step).  transposed=(r0, r1): the split of W^T[r0:r1, :] instead -- the operand of dx = dy . W for input
    columns r0..r1.  bf16=True (default: inside a `bf16_compute` scope): the bf16 form (w, None, n_pad, rows) instead, w
    [n_pad, k_pad] torch.bfloat16 rounded to nearest even, cached separately."""
    if torch.is_tensor(weights):
        weights = (weights,)
    bf16 = bf16_compute_active() if bf16 is None else bool(bf16)
    # keyed by the identity of the source tensor OBJECTS (validated through weak references and version counters):
    # a data_ptr key would go stale when the allocator hands a freed weight's address to a new tensor
    key = tuple(id(w) for w in weights) + (col0, cols, k_pad, kcat, transposed, bf16)
    hit = _TC_WEIGHTS.get(key)
    if hit is not None:
        refs, versions, ptrs, result = hit
        if all(r() is w and w._version == v and w.data_ptr() == p for r, w, v, p in zip(refs, weights, versions, ptrs)):
            return result
    _TLS.unsettled = 3   # the split below writes what the next tensor-core launches read: see tc_linear()
    mats = [w.detach().reshape(w.shape[0], -1) for w in weights]
    if transposed is not None:
        mats = [m.t()[transposed[0]:transposed[1]].contiguous() for m in mats]
    if kcat:   # [W_a | W_b | ...] along K: one GEMM over concatenated sources adds the layers' outputs
        mats = [torch.cat(mats, 1).contiguous()]
    ld = mats[0].shape[1]
    ncols = ld - col0 if cols is None else cols
    kp = (ncols + 31) // 32 * 32 if k_pad is None else k_pad
    rows = sum(m.shape[0] for m in mats)
    n_pad = (rows + 15) // 16 * 16
    # (the split kernel writes every entry of the rows it is given, padding columns included: zero-fill only for padding rows)
    alloc = torch.empty if n_pad == rows else torch.zeros
    if bf16:
        hi, lo = alloc(n_pad, kp, dtype=torch.bfloat16, device=mats[0].device), None
    else:
        hi = alloc(n_pad, kp, dtype=torch.float32, device=mats[0].device)
        lo = alloc(n_pad, kp, dtype=torch.float32, device=mats[0].device)
    r0 = 0
    for m in mats:
        if bf16:
            check(lib().pvraft_tc_weight_bf16(_p(m.contiguous()), m.shape[0], ncols, ld, col0, m.shape[0], kp, hi[r0:].data_ptr(),
                                              _stream()), 'tc_weight_bf16')
        else:
            check(lib().pvraft_tc_weight_split(_p(m.contiguous()), m.shape[0], ncols, ld, col0, m.shape[0], kp,
                                               hi[r0:].data_ptr(), lo[r0:].data_ptr(), _stream()), 'tc_weight_split')
        r0 += m.shape[0]
    if len(_TC_WEIGHTS) > 512:
        _TC_WEIGHTS.clear()
    result = (hi, lo, n_pad, rows)
    _TC_WEIGHTS[key] = (tuple(weakref.ref(w) for w in weights), tuple(w._version for w in weights),
                        tuple(w.data_ptr() for w in weights), result)
    return result


_DERIVED = {}


def derived(tensors, tag, fn):
    """Cache of small host- or device-side values derived from parameters (a bias sum, a PReLU slope read back once);
    keyed by parameter identity, re-derived when a parameter's version or storage changes."""
    key = tuple(id(t) for t in tensors) + (tag,)
    hit = _DERIVED.get(key)
    if hit is not None:
        refs, versions, ptrs, value = hit
        if all(r() is t and t._version == v and t.data_ptr() == p for r, t, v, p in zip(refs, tensors, versions, ptrs)):
            return value
    _TLS.unsettled = 3   # fn may launch kernels that write a folded weight / bias
    value = fn(*tensors)
    if len(_DERIVED) > 512:
        _DERIVED.clear()
    _DERIVED[key] = (tuple(weakref.ref(t) for t in tensors), tuple(t._version for t in tensors),
                     tuple(t.data_ptr() for t in tensors), value)
    return value


KNN_SORT_MAX_N = 16384   # largest cloud the kNN grid sorts in shared memory (csrc/knn.cu); beyond it a counting sort builds the grid


def point_order(points):
    """[B,N,3] -> [B,N] int32: Morton order over the cells of the kNN grid, from the library's in-shared-memory sort
    (one launch; the torch formulation below costs ~40 launches)."""
    b, n, _ = points.shape
    ws_bytes = int(lib().pvraft_knn_workspace_bytes(b, n))
    if ws_bytes <= 0 or n < 64 or n > KNN_SORT_MAX_N:
        return morton_order(points).to(torch.int32).contiguous()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=points.device)
    perm = torch.empty(b, n, dtype=torch.int32, device=points.device)
    _count(lib().pvraft_point_order_fwd(_p(points), b, n, _p(perm, torch.int32), _p(ws, torch.uint8), _stream()), 'point_order')
    return perm


def morton_order(points):
    """[B,N,3] -> [B,N] int64 permutation that sorts every cloud along a 30-bit Morton (Z-order) curve: neighbouring points
    get neighbouring rows, so the 32 neighbour rows a SetConv gathers for consecutive points overlap in L1/L2."""
    lo, hi = points.amin(1, keepdim=True), points.amax(1, keepdim=True)
    q = ((points - lo) / (hi - lo).clamp_min(1e-12) * 1023.0).long().clamp_(0, 1023)

    def spread(v):   # 10 bits -> every third bit
        v = (v | (v << 16)) & 0x030000FF
        v = (v | (v << 8)) & 0x0300F00F
        v = (v | (v << 4)) & 0x030C30C3
        return (v | (v << 2)) & 0x09249249

    code = spread(q[..., 0]) | (spread(q[..., 1]) << 1) | (spread(q[..., 2]) << 2)
    return torch.sort(code, dim=1, stable=True).indices


def tc_supported(n_points, *channels):
    """The tensor-core layer needs 128-point tiles that do not straddle samples and 32-channel k-blocks."""
    return n_points % 128 == 0 and all(c % 32 == 0 for c in channels)


def tc_linear(sources, w, bias=None, *, in_min=None, in_stats=None, in_gamma=None, in_beta=None, in_count=0.0,
              in_act=ACT_NONE, in_slope=0.0, out_act=ACT_NONE, residual=None, out=None, out_stats=None, epilogue=TC_PLAIN,
              bias2=None, out2=None, h=None, z=None, cout=None, tail=None, w3=None, b3=None, coords1=None, coords2=None,
              coords2_out=None, flow_out=None):
    """Fused layer on the Hopper tensor cores (wgmma).  sources: list of [B,N,C_i] tensors concatenated along K (the
    GroupNorm prologue applies to sources[0]); w = (hi, lo, n_pad, rows) from tc_weights() -- its bf16 form runs the layer on
    bf16 operands; tail [B,N,3] fills the output columns cout..cout+2."""
    hi, lo, n_pad, rows = w
    b, n, _ = sources[0].shape
    cout = rows if cout is None else cout
    if out is None:
        out = torch.empty(b, n, cout + (3 if tail is not None else 0), dtype=torch.float32, device=sources[0].device)
    a = _lib.TcLinearArgs()
    for i, src in enumerate(sources):
        a.in_[i] = _p(src)
        a.in_channels[i] = src.shape[-1]
    a.in_min, a.in_stats, a.in_gamma, a.in_beta = _p(in_min), _p(in_stats, torch.float64), _p(in_gamma), _p(in_beta)
    a.in_count, a.in_act, a.in_slope = float(in_count), in_act, float(in_slope)
    if lo is None:
        a.w_bf16 = _p(hi, torch.bfloat16)
    else:
        a.w_hi, a.w_lo = _p(hi), _p(lo)
    a.n_pad, a.cout = n_pad, cout
    a.bias, a.bias2, a.out_act, a.residual = _p(bias), _p(bias2), out_act, _p(residual)
    a.out, a.out2, a.h, a.z = _p(out), _p(out2), _p(h), _p(z)
    a.out_stats, a.epilogue, a.B, a.N = _p(out_stats, torch.float64), epilogue, b, n
    a.tail = _p(tail)
    a.w3, a.b3, a.coords1, a.coords2 = _p(w3), _p(b3), _p(coords1), _p(coords2)
    a.coords2_out, a.flow_out = _p(coords2_out), _p(flow_out)
    # The kernel may fetch its parameters while the previous kernel drains (PDL) once they are settled: not during the
    # three tensor-core launches that follow a weight split or a re-derived folded parameter on this thread.
    pending = getattr(_TLS, 'unsettled', 0)
    a.params_settled = 1 if pending == 0 else 0
    if pending:
        _TLS.unsettled = pending - 1
    ws = _det_workspace(lib().pvraft_tc_linear_det_workspace_bytes, b, device=out.device) if out_stats is not None else None
    _count(lib().pvraft_tc_linear_fwd(C.byref(a), _p(ws, torch.uint8), _stream()), 'tc_linear')
    return out


fuse_update_chain = True   # False: the RAFT loop runs the update chain as its five tc_linear launches (tests compare the two)


def update_chain(y1, gn, kfeat, cflow, flow, net, inp, weights, biases):
    """MotionEncoder + ConvGRU + flow-head fc1 pre-transform of one RAFT iteration in one launch (include/pvraft_b200.h,
    pvraft_update_chain_fwd): the same bits as the five tc_linear launches it replaces.  gn: y1's prologue (in_stats,
    in_gamma, in_beta, in_count, in_slope as for tc_linear); weights: five tc_weights() results in the order cc, motion,
    [z|r], q, fc1, all five in the 3xTF32 or all five in the bf16 form; biases: (b_cc, b_m, b_z, b_r, b_q).
    Returns (net' [B,N,64], P [B,N,64])."""
    b, n, _ = net.shape
    net_out, p_out = torch.empty_like(net), torch.empty_like(net)
    a = _lib.UpdateChainArgs()
    a.y1, a.y1_stats = _p(y1), _p(gn['in_stats'], torch.float64)
    a.gn_gamma, a.gn_beta, a.gn_count, a.gn_slope = _p(gn['in_gamma']), _p(gn['in_beta']), float(gn['in_count']), float(gn['in_slope'])
    a.kfeat, a.cflow, a.flow, a.net, a.inp = _p(kfeat), _p(cflow), _p(flow), _p(net), _p(inp)
    for i, (hi, lo, _, _) in enumerate(weights):
        if lo is None:
            a.w_bf16[i] = _p(hi, torch.bfloat16)
        else:
            a.w_hi[i], a.w_lo[i] = _p(hi), _p(lo)
    a.b_cc, a.b_m, a.b_z, a.b_r, a.b_q = (_p(x) for x in biases)
    a.net_out, a.p_out = _p(net_out), _p(p_out)
    a.B, a.N, a.hidden, a.context, a.y1_channels = b, n, net.shape[-1], inp.shape[-1], y1.shape[-1]
    _count(lib().pvraft_update_chain_fwd(C.byref(a), _stream()), 'update_chain')
    return net_out, p_out


def gn_act(x, stats, gamma, beta, count, act=ACT_LRELU, slope=0.1, transpose_out=False, slope_dev=None):
    """slope_dev: optional one-element device tensor (a PReLU weight) the kernel reads instead of the scalar `slope`."""
    b, n, c = x.shape
    out = torch.empty((b, c, n) if transpose_out else (b, n, c), dtype=torch.float32, device=x.device)
    _count(lib().pvraft_gn_act_fwd(_p(x), _p(stats, torch.float64), _p(gamma), _p(beta), float(count), act, float(slope),
                                   b, n, c, int(transpose_out), _p(out), _p(slope_dev), _stream()), 'gn_act')
    return out


def transpose(x):
    """[B,R,C] -> [B,C,R] contiguous."""
    b, r, c = x.shape
    out = torch.empty(b, c, r, dtype=torch.float32, device=x.device)
    _count(lib().pvraft_transpose_fwd(_p(x), b, r, c, _p(out), _stream()), 'transpose')
    return out


def corr_feature(args):
    _count(lib().pvraft_corr_feature_fwd(C.byref(args), _stream()), 'corr_feature')


def knn_branch(args):
    _count(lib().pvraft_knn_branch_fwd(C.byref(args), _stream()), 'knn_branch')


def gru(args):
    _count(lib().pvraft_gru_fwd(C.byref(args), _stream()), 'gru')


def flow_out(args):
    _count(lib().pvraft_flow_out_fwd(C.byref(args), _stream()), 'flow_out')


def edge_plan(nbr, order=None):
    """The SetConv edge kernel's gather plan of the kNN graph nbr [B,N,32] processed in `order` ([B,N] or None):
    uint8 [B, tiles per sample, record bytes], sample-major, so plan[:b] is the plan of nbr[:b] (csrc/edge_plan.cuh)."""
    b, n, _ = nbr.shape
    rec = int(lib().pvraft_edge_plan_bytes(1, 1))
    tiles = int(lib().pvraft_edge_plan_bytes(1, n)) // rec
    plan = torch.empty(b, tiles, rec, dtype=torch.uint8, device=nbr.device)
    _count(lib().pvraft_edge_plan_fwd(_p(nbr, torch.int32), _p(order, torch.int32), b, n, _p(plan, torch.uint8), _stream()),
           'edge_plan')
    return plan


def setconv_edge(fc1p, nbr, edge_feats, w_fc1, cin, stats, ymax=None, ymin=None, order=None, plan=None):
    """plan: edge_plan(nbr, order), built here when not given (a Graph keeps its own)."""
    b, n, c = fc1p.shape
    if ymax is None:
        ymax = torch.empty_like(fc1p)
    if ymin is None:
        ymin = torch.empty_like(fc1p)
    if plan is None:
        plan = edge_plan(nbr, order)
    elif plan.shape[0] != b or plan.numel() != int(lib().pvraft_edge_plan_bytes(b, n)):
        raise ValueError(f'edge plan of shape {tuple(plan.shape)} does not belong to a graph of {b} x {n} points')
    ws = _det_workspace(lib().pvraft_setconv_edge_det_workspace_bytes, b, device=fc1p.device)
    _count(lib().pvraft_setconv_edge_fwd(_p(fc1p), _p(nbr, torch.int32), _p(edge_feats), _p(w_fc1), cin, b, n, c, _p(ymax), _p(ymin),
                                         _p(stats, torch.float64), _p(order, torch.int32), _p(plan, torch.uint8), _p(ws, torch.uint8),
                                         _stream()), 'setconv_edge')
    return ymax, ymin


def knn(xyz, query, k, mode=0, want_rel=False, use_sweep=True):
    """-> int32 [B,S,k] local ids of the k nearest `xyz` points of every query (unordered)
    [, rel [B,S,k,3] = xyz[idx] - query]."""
    b, n, _ = xyz.shape
    s = query.shape[1]
    out = torch.empty(b, s, k, dtype=torch.int32, device=xyz.device)
    rel = torch.empty(b, s, k, 3, dtype=torch.float32, device=xyz.device) if want_rel else None
    ws_bytes = int(lib().pvraft_knn_workspace_bytes(b, n)) if use_sweep else 0
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=xyz.device) if ws_bytes > 0 else None
    _count(lib().pvraft_knn_fwd(_p(xyz), _p(query), b, n, s, k, mode, _p(out, torch.int32), _p(rel),
                                _p(ws, torch.uint8), _stream()), 'knn')
    return (out, rel) if want_rel else out


# ---- gradient contract (include/pvraft_b200.h, "Gradient contract"): thin wrappers used by pvraft_b200/train.py ------------
def linear_wgrad(x, dy, dw, db=None):
    """dw [cout,cin] += dy^T x, db [cout] += column sums of dy (both zeroed by the caller); x [B,R,cin], dy [B,R,cout]."""
    rows = x.shape[0] * x.shape[1]
    ws = _det_workspace(lib().pvraft_linear_wgrad_det_workspace_bytes, x.shape[-1], dy.shape[-1], device=x.device)
    _count(lib().pvraft_linear_wgrad(_p(x), _p(dy), rows, x.shape[-1], dy.shape[-1], _p(dw), dw.shape[-1], _p(db), _p(ws, torch.uint8),
                                     _stream()), 'linear_wgrad')


def tc_wgrad_bf16(x, dy, dw, db=None):
    """linear_wgrad on the tensor cores with bf16 operands (round to nearest even, fp32 accumulation): dw [cout,cin] +=
    bf16(dy)^T bf16(x), db [cout] += column sums of the unrounded dy; x [B,R,cin], dy [B,R,cout], cin in {32..192} and
    cout in {32..128} multiples of 32."""
    rows = x.shape[0] * x.shape[1]
    ws = _det_workspace(lib().pvraft_tc_wgrad_bf16_det_workspace_bytes, x.shape[-1], dy.shape[-1], device=x.device)
    _count(lib().pvraft_tc_wgrad_bf16(_p(x), _p(dy), rows, x.shape[-1], dy.shape[-1], _p(dw), dw.shape[-1], _p(db), _p(ws, torch.uint8),
                                      _stream()), 'tc_wgrad_bf16')


def linear_bwd_small(x, dy, w, dw, db=None, want_dx=False):
    """cin <= 4, cout in {16,32,48,64,96,128}: dw += dy^T x, db += column sums, and dx = dy w (returned, or None) in one pass over dy."""
    rows = x.shape[0] * x.shape[1]
    dx = torch.empty_like(x) if want_dx else None
    ws = _det_workspace(lib().pvraft_linear_bwd_small_det_workspace_bytes, x.shape[-1], dy.shape[-1], device=x.device)
    _count(lib().pvraft_linear_bwd_small(_p(x), _p(dy), _p(w), rows, x.shape[-1], dy.shape[-1], w.shape[-1], _p(dw), dw.shape[-1], _p(db),
                                         _p(dx), _p(ws, torch.uint8), _stream()), 'linear_bwd_small')
    return dx


def gn_act_maxk(x, stats, gamma, beta, count, act, slope, slope_dev=None):
    """x [B, pts*32, C] -> (max over each point's 32 rows of act(GN(x)) [B,pts,C], arg uint8 [B,pts,C]), one pass."""
    b, rows, c = x.shape
    y = torch.empty(b, rows // 32, c, dtype=torch.float32, device=x.device)
    arg = torch.empty(b, rows // 32, c, dtype=torch.uint8, device=x.device)
    _count(lib().pvraft_gn_act_maxk_fwd(_p(x), _p(stats, torch.float64), _p(gamma), _p(beta), float(count), act, float(slope), b,
                                        rows // 32, c, _p(y), _p(arg, torch.uint8), _p(slope_dev), _stream()), 'gn_act_maxk')
    return y, arg


def gn_act_bwd(x, dy, stats, gamma, beta, count, act, slope, want_dslope=False, slope_dev=None, arg=None):
    """-> (dx, dgamma [C] f32, dbeta [C] f32, dslope [1] f32 or None)."""
    b, rows, c = x.shape
    dev = x.device
    scratch = torch.zeros(b * 16 + 2 * c + 1, dtype=torch.float64, device=dev)   # gsum | dgamma | dbeta | dslope
    gsum, dgamma, dbeta, dslope = scratch[:b * 16], scratch[b * 16:b * 16 + c], scratch[b * 16 + c:b * 16 + 2 * c], scratch[-1:]
    dx = torch.empty_like(x)
    ws = _det_workspace(lib().pvraft_gn_act_bwd_det_workspace_bytes, b, c, device=dev)
    _count(lib().pvraft_gn_act_bwd(_p(x), _p(dy), _p(stats, torch.float64), _p(gamma), _p(beta), float(count), act, float(slope), b, rows, c,
                                   gsum.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), dslope.data_ptr() if want_dslope else None, _p(dx),
                                   _p(slope_dev), _p(arg, torch.uint8), _p(ws, torch.uint8), _stream()), 'gn_act_bwd')
    return dx, dgamma.float(), dbeta.float(), (dslope.float() if want_dslope else None)


def edge_fwd(p, nbr, e, stats=None):
    """e [B,N*32,C] <- p[nbr] - p[centre] + e in place; stats [B,8,2] f64 accumulated."""
    b, n, c = p.shape
    ws = _det_workspace(lib().pvraft_edge_fwd_det_workspace_bytes, b, device=p.device) if stats is not None else None
    _count(lib().pvraft_edge_fwd(_p(p), _p(nbr, torch.int32), _p(e), b, n, c, _p(stats, torch.float64), _p(ws, torch.uint8), _stream()),
           'edge_fwd')
    return e


def edge_bwd(dt, nbr, dp):
    b, n, c = dp.shape
    ws = _det_workspace(lib().pvraft_edge_bwd_det_workspace_bytes, b, n, c, device=dp.device)
    _count(lib().pvraft_edge_bwd(_p(dt), _p(nbr, torch.int32), b, n, c, _p(dp), _p(ws, torch.uint8), _stream()), 'edge_bwd')
    return dp


def maxk_fwd(x, pts, c):
    y = torch.empty(pts, c, dtype=torch.float32, device=x.device)
    arg = torch.empty(pts, c, dtype=torch.uint8, device=x.device)
    _count(lib().pvraft_maxk_fwd(_p(x), pts, c, _p(y), _p(arg, torch.uint8), _stream()), 'maxk_fwd')
    return y, arg


def maxk_bwd(dy, arg, pts, c):
    dx = torch.empty(pts, KNN, c, dtype=torch.float32, device=dy.device)
    _count(lib().pvraft_maxk_bwd(_p(dy), _p(arg, torch.uint8), pts, c, _p(dx), _stream()), 'maxk_bwd')
    return dx


def lookup_table_in_smem(m, k):
    """True when corr_lookup stages the gather table of a second cloud of m points in shared memory at truncate_k = k (the
    faster path).  At K = 512 a table of 8 192 points fits and one of 12 000 does not: the kernel then gathers from global
    memory."""
    return bool(lib().pvraft_corr_lookup_table_in_smem(int(m), int(k)))


def corr_lookup_bwd(corr_idx, xyz2_pad, coords, slots, g_vox, g_sel, levels, base_scale):
    """-> d_corr [B,N,K]; the state's ids are rows of the gather table xyz2_pad [B,M,4]."""
    b, n, k = corr_idx.shape
    m = _table_rows(xyz2_pad, b)
    d_corr = torch.empty(b, n, k, dtype=torch.float32, device=corr_idx.device)
    _count(lib().pvraft_corr_lookup_bwd(_p(corr_idx, torch.int32), _p(xyz2_pad), _p(coords), _p(slots, torch.int32), _p(g_vox),
                                        g_vox.shape[-1], _p(g_sel), b, n, m, k, levels, float(base_scale), _p(d_corr), _stream()),
           'corr_lookup_bwd')
    return d_corr


def corr_lookup_xyz_bwd(corr_idx, slots, g_sel, d_xyz2):
    """d_xyz2 [B,M,3] (zeroed by the caller) += the gradient of the kNN 4-vectors g_sel [B,N*32,4] w.r.t. the second cloud's
    rows, through the state's ids corr_idx [B,N,K] and the forward's slots [B,N,32]."""
    b, n, k = corr_idx.shape
    m = d_xyz2.shape[1]
    ws = _det_workspace(lib().pvraft_corr_lookup_xyz_bwd_det_workspace_bytes, b, m, device=d_xyz2.device)
    _count(lib().pvraft_corr_lookup_xyz_bwd(_p(corr_idx, torch.int32), _p(slots, torch.int32), _p(g_sel), b, n, m, k, _p(d_xyz2),
                                            _p(ws, torch.uint8), _stream()), 'corr_lookup_xyz_bwd')
    return d_xyz2


def corr_init_bwd(g, idx, fmap1, fmap2):
    """g, idx [B,N,K], fmap1 [B,N,C], fmap2 [B,M,C] -> (d fmap1 [B,N,C], d fmap2 [B,M,C])."""
    b, n, c = fmap1.shape
    m = fmap2.shape[1]
    if fmap2.shape != (b, m, c):
        raise ValueError(f'corr_init_bwd: feature maps {tuple(fmap1.shape)} and {tuple(fmap2.shape)}')
    d1 = torch.empty_like(fmap1)
    d2 = torch.zeros_like(fmap2)
    ws = _det_workspace(lib().pvraft_corr_init_bwd_det_workspace_bytes, b, m, c, device=fmap1.device)
    _count(lib().pvraft_corr_init_bwd(_p(g), _p(idx, torch.int32), _p(fmap1), _p(fmap2), b, n, m, c, g.shape[-1], _p(d1), _p(d2),
                                      _p(ws, torch.uint8), _stream()), 'corr_init_bwd')
    return d1, d2


def _loss_batch(what, x, b_rows, m=None):
    """The shape rules of the self-supervised loss kernels: x [S,N,3] with S a multiple of the batch size b_rows."""
    if x.dim() != 3 or x.shape[-1] != 3 or x.shape[0] < 1 or x.shape[1] < 1:
        raise ValueError(f'{what}: expected [S,N,3], got {tuple(x.shape)}')
    if b_rows < 1 or x.shape[0] % b_rows:
        raise ValueError(f'{what}: {x.shape[0]} samples are not a whole number of batches of {b_rows}')
    if m is not None and m < 1:
        raise ValueError(f'{what}: the second cloud is empty')


# Per op, searched clouds of at least this many points are searched on a uniform-grid index (pvraft_*_grid_fwd) instead of by
# brute force.  Both forms return the same neighbours in the same order, so the choice only changes the time.  Measured with
# tools/grid_search_cost.py on an H100 80GB HBM3 at 700 W (DESIGN.md 4.4): at N = M = 8192 the grid form of Chamfer (S = 8)
# and of the Laplacian term take 0.52 / 0.42 ms against 0.54 / 0.60 ms, while the propagation (B = 1, k = 3) takes 0.24 ms
# against 0.12 ms; at 32 768 every grid form is at least 2x faster.  flow_consistency runs the Laplacian's search and takes
# its threshold (DESIGN.md 4.8).
GRID_SEARCH_MIN_POINTS = {'chamfer': 8192, 'laplacian': 8192, 'flow_propagate': 32768}


def use_grid_search(op, searched, use_grid=None):
    """True when the nearest-neighbour op `op` ('chamfer', 'laplacian', 'flow_propagate') runs its grid form for a searched
    cloud of `searched` points.  `use_grid` True / False forces the grid / brute-force form; it exists for tests and
    measurement, and the models and losses leave it None."""
    if use_grid is not None:
        return bool(use_grid)
    return searched >= GRID_SEARCH_MIN_POINTS[op]


def _workspace(nbytes, device):
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)


def chamfer(a, b, use_grid=None):
    """a [S,N,3] (the first clouds moved by the flows), b [B,M,3] (the second clouds; sample s searches b[s % B]) ->
    (acc [S,2] f64: the sums over a's points of their least squared distance to b, and over b's points of theirs to a;
    nn_ab [S,N] int32, nn_ba [S,M] int32: the nearest points, lowest index on ties).  Both directions in one launch.
    The grid form runs when the larger cloud has GRID_SEARCH_MIN_POINTS['chamfer'] points (`use_grid`: see use_grid_search)."""
    if b.dim() != 3 or b.shape[-1] != 3:
        raise ValueError(f'chamfer: expected b [B,M,3], got {tuple(b.shape)}')
    s, n, _ = a.shape
    bb, m = int(b.shape[0]), int(b.shape[1])
    _loss_batch('chamfer', a, bb, m)
    acc = torch.zeros(s, 2, dtype=torch.float64, device=a.device)
    nn_ab = torch.empty(s, n, dtype=torch.int32, device=a.device)
    nn_ba = torch.empty(s, m, dtype=torch.int32, device=a.device)
    ws = _det_workspace(lib().pvraft_chamfer_fwd_det_workspace_bytes, s, device=a.device)
    if use_grid_search('chamfer', max(n, m), use_grid):
        gw = _workspace(lib().pvraft_chamfer_grid_workspace_bytes(s, bb, n, m), a.device)
        _count(lib().pvraft_chamfer_grid_fwd(_p(a), _p(b), s, bb, n, m, _p(nn_ab, torch.int32), _p(nn_ba, torch.int32), _p(acc, torch.float64),
                                             _p(gw, torch.uint8), _p(ws, torch.uint8), _stream()), 'chamfer_grid_fwd')
        return acc, nn_ab, nn_ba
    _count(lib().pvraft_chamfer_fwd(_p(a), _p(b), s, bb, n, m, _p(nn_ab, torch.int32), _p(nn_ba, torch.int32), _p(acc, torch.float64),
                                    _p(ws, torch.uint8), _stream()), 'chamfer_fwd')
    return acc, nn_ab, nn_ba


def chamfer_bwd(a, b, nn_ab, nn_ba, g, want_db=True):
    """Gradients of C_s = acc[s,0]/N + acc[s,1]/M (chamfer) with the indices held fixed, for the upstream gradient g [S]
    (on the device) -> (d_a [S,N,3], d_b [B,M,3] or None)."""
    s, n, _ = a.shape
    bb, m = int(b.shape[0]), int(b.shape[1])
    _loss_batch('chamfer_bwd', a, bb, m)
    if g.shape != (s,):
        raise ValueError(f'chamfer_bwd: expected g [{s}], got {tuple(g.shape)}')
    d_a = torch.zeros_like(a)
    d_b = torch.zeros_like(b) if want_db else None
    ws = _det_workspace(lib().pvraft_chamfer_bwd_det_workspace_bytes, s, bb, n, m, device=a.device)
    _count(lib().pvraft_chamfer_bwd(_p(a), _p(b), _p(nn_ab, torch.int32), _p(nn_ba, torch.int32), _p(g), s, bb, n, m, _p(d_a), _p(d_b),
                                    _p(ws, torch.uint8), _stream()), 'chamfer_bwd')
    return d_a, d_b


def _smooth_args(what, f, nbr):
    if nbr.dim() != 3 or nbr.shape[1] != f.shape[1] or not 1 <= nbr.shape[2] <= KNN:
        raise ValueError(f'{what}: expected nbr [B,{f.shape[1]},k] with 1 <= k <= {KNN}, got {tuple(nbr.shape)}')
    _loss_batch(what, f, int(nbr.shape[0]))
    return f.shape[0], int(nbr.shape[0]), f.shape[1], int(nbr.shape[2])


def flow_smooth(f, nbr):
    """f [S,N,3], nbr [B,N,k] int32 (sample s uses nbr[s % B]) -> acc [S] f64: sum over the edges of ||f_j - f_i||."""
    s, bb, n, k = _smooth_args('flow_smooth', f, nbr)
    acc = torch.zeros(s, dtype=torch.float64, device=f.device)
    ws = _det_workspace(lib().pvraft_flow_smooth_fwd_det_workspace_bytes, s, device=f.device)
    _count(lib().pvraft_flow_smooth_fwd(_p(f), _p(nbr, torch.int32), s, bb, n, k, _p(acc, torch.float64), _p(ws, torch.uint8), _stream()),
           'flow_smooth_fwd')
    return acc


def flow_smooth_bwd(f, nbr, g):
    """Gradient of S_s = acc[s] / (N k) (flow_smooth) for the upstream gradient g [S] (on the device) -> d_f [S,N,3]."""
    s, bb, n, k = _smooth_args('flow_smooth_bwd', f, nbr)
    if g.shape != (s,):
        raise ValueError(f'flow_smooth_bwd: expected g [{s}], got {tuple(g.shape)}')
    d_f = torch.zeros_like(f)
    ws = _det_workspace(lib().pvraft_flow_smooth_bwd_det_workspace_bytes, s, n, device=f.device)
    _count(lib().pvraft_flow_smooth_bwd(_p(f), _p(nbr, torch.int32), _p(g), s, bb, n, k, _p(d_f), _p(ws, torch.uint8), _stream()),
           'flow_smooth_bwd')
    return d_f


LAPLACIAN_MAX_K_INT = 8   # neighbours pvraft_laplacian_fwd interpolates from at most


def _graph_args(what, x, nbr):
    """x [B,N,3], nbr [B,N,k] int32 with 2 <= k <= min(32, N): the rules of the Laplacian graphs."""
    if x.dim() != 3 or x.shape[-1] != 3 or x.shape[0] < 1 or x.shape[1] < 1:
        raise ValueError(f'{what}: expected [B,N,3], got {tuple(x.shape)}')
    if nbr.dim() != 3 or tuple(nbr.shape[:2]) != tuple(x.shape[:2]) or not 2 <= nbr.shape[2] <= min(KNN, x.shape[1]):
        raise ValueError(f'{what}: expected nbr [{x.shape[0]},{x.shape[1]},k] with 2 <= k <= min({KNN}, N), got {tuple(nbr.shape)}')
    return int(x.shape[0]), int(x.shape[1]), int(nbr.shape[2])


def cloud_laplacian(x, nbr):
    """x [B,N,3], nbr [B,N,k] int32 (a kNN graph that includes each point) -> L(x) [B,N,3],
    L(x)_i = sum_e (x[nbr[i,e]] - x_i) / (k - 1)."""
    b, n, k = _graph_args('cloud_laplacian', x, nbr)
    out = torch.empty_like(x)
    _count(lib().pvraft_cloud_laplacian_fwd(_p(x), _p(nbr, torch.int32), b, n, k, _p(out), _stream()), 'cloud_laplacian_fwd')
    return out


def cloud_laplacian_bwd(g_l, nbr, d_x):
    """d_x [B,N,3] += the gradient of L(x) (cloud_laplacian) for the upstream gradient g_l [B,N,3]; returns d_x."""
    b, n, k = _graph_args('cloud_laplacian_bwd', g_l, nbr)
    if d_x.shape != g_l.shape:
        raise ValueError(f'cloud_laplacian_bwd: d_x {tuple(d_x.shape)} does not match g_l {tuple(g_l.shape)}')
    ws = _det_workspace(lib().pvraft_cloud_laplacian_bwd_det_workspace_bytes, b, n, device=g_l.device)
    _count(lib().pvraft_cloud_laplacian_bwd(_p(g_l), _p(nbr, torch.int32), b, n, k, _p(d_x), _p(ws, torch.uint8), _stream()),
           'cloud_laplacian_bwd')
    return d_x


def _laplacian_args(what, w, p2, l2, g1, k_int):
    if p2.dim() != 3 or p2.shape[-1] != 3 or l2.shape != p2.shape:
        raise ValueError(f'{what}: expected p2 and l2 [B,M,3], got {tuple(p2.shape)} and {tuple(l2.shape)}')
    bb, m = int(p2.shape[0]), int(p2.shape[1])
    _loss_batch(what, w, bb, m)
    s, n = int(w.shape[0]), int(w.shape[1])
    if g1.dim() != 3 or tuple(g1.shape[:2]) != (bb, n) or not 2 <= g1.shape[2] <= min(KNN, n):
        raise ValueError(f'{what}: expected g1 [{bb},{n},k_lap] with 2 <= k_lap <= min({KNN}, N), got {tuple(g1.shape)}')
    if isinstance(k_int, bool) or not isinstance(k_int, int) or not 1 <= k_int <= min(LAPLACIAN_MAX_K_INT, m):
        raise ValueError(f'{what}: k_int={k_int!r} must be an integer in 1..min({LAPLACIAN_MAX_K_INT}, M={m})')
    return s, bb, n, m, int(g1.shape[2])


def laplacian(w, p2, l2, g1, k_int, use_grid=None):
    """w [S,N,3] (the first clouds moved by the flows), p2 [B,M,3] and its Laplacian l2 = cloud_laplacian(p2, g2), g1 [B,N,k_lap]
    (the first cloud's graph; sample s uses entry s % B) -> (acc [S] f64: sum_i ||Lhat_i - L(w)_i||^2 with Lhat_i the
    inverse-squared-distance interpolation of l2 over the k_int nearest points of p2; nn_idx [S,N,k_int] int32, nearest first,
    lowest index on ties; res [S,N,3] = Lhat - L(w)).  R_s = acc[s] / N.  The grid form runs when p2 has
    GRID_SEARCH_MIN_POINTS['laplacian'] points (`use_grid`: see use_grid_search)."""
    s, bb, n, m, kl = _laplacian_args('laplacian', w, p2, l2, g1, k_int)
    acc = torch.zeros(s, dtype=torch.float64, device=w.device)
    nn_idx = torch.empty(s, n, k_int, dtype=torch.int32, device=w.device)
    res = torch.empty_like(w)
    ws = _det_workspace(lib().pvraft_laplacian_fwd_det_workspace_bytes, s, device=w.device)
    if use_grid_search('laplacian', m, use_grid):
        gw = _workspace(lib().pvraft_grid_index_workspace_bytes(bb, m), w.device)
        _count(lib().pvraft_laplacian_grid_fwd(_p(w), _p(p2), _p(l2), _p(g1, torch.int32), s, bb, n, m, kl, k_int, _p(nn_idx, torch.int32),
                                               _p(res), _p(acc, torch.float64), _p(gw, torch.uint8), _p(ws, torch.uint8), _stream()),
               'laplacian_grid_fwd')
        return acc, nn_idx, res
    _count(lib().pvraft_laplacian_fwd(_p(w), _p(p2), _p(l2), _p(g1, torch.int32), s, bb, n, m, kl, k_int, _p(nn_idx, torch.int32), _p(res),
                                      _p(acc, torch.float64), _p(ws, torch.uint8), _stream()), 'laplacian_fwd')
    return acc, nn_idx, res


def laplacian_bwd(w, p2, l2, g1, nn_idx, res, g, want_dp2=True):
    """Gradients of R_s = acc[s] / N (laplacian) with nn_idx held fixed, for the upstream gradient g [S] (on the device) ->
    (d_w [S,N,3], d_p2 [B,M,3] (the distance part; None unless want_dp2), d_l2 [B,M,3] (None unless want_dp2)).  d_l2 reaches p2
    through cloud_laplacian_bwd."""
    s, bb, n, m, kl = _laplacian_args('laplacian_bwd', w, p2, l2, g1, int(nn_idx.shape[-1]) if nn_idx.dim() == 3 else -1)
    if tuple(nn_idx.shape[:2]) != (s, n) or res.shape != w.shape:
        raise ValueError(f'laplacian_bwd: nn_idx {tuple(nn_idx.shape)} and res {tuple(res.shape)} do not match w {tuple(w.shape)}')
    if g.shape != (s,):
        raise ValueError(f'laplacian_bwd: expected g [{s}], got {tuple(g.shape)}')
    d_w = torch.zeros_like(w)
    d_p2 = torch.zeros_like(p2) if want_dp2 else None
    d_l2 = torch.zeros_like(p2) if want_dp2 else None
    ws = _det_workspace(lib().pvraft_laplacian_bwd_det_workspace_bytes, s, bb, n, m, device=w.device)
    _count(lib().pvraft_laplacian_bwd(_p(w), _p(p2), _p(l2), _p(g1, torch.int32), _p(nn_idx, torch.int32), _p(res), _p(g), s, bb, n, m, kl,
                                      int(nn_idx.shape[-1]), _p(d_w), _p(d_p2), _p(d_l2), _p(ws, torch.uint8), _stream()), 'laplacian_bwd')
    return d_w, d_p2, d_l2


CONSISTENCY_MAX_K = 8   # neighbours pvraft_flow_consistency_fwd interpolates the reverse flow from at most


def _consistency_args(what, w, p2, f21, k, n_f12=None):
    if p2.dim() != 3 or p2.shape[-1] != 3:
        raise ValueError(f'{what}: expected p2 [B,M,3], got {tuple(p2.shape)}')
    bb, m = int(p2.shape[0]), int(p2.shape[1])
    _loss_batch(what, w, bb, m)
    s, n = int(w.shape[0]), int(w.shape[1])
    if f21.dim() != 3 or tuple(f21.shape) != (s, m, 3):
        raise ValueError(f'{what}: expected f21 [{s},{m},3], got {tuple(f21.shape)}')
    if n_f12 is not None and tuple(n_f12.shape) != tuple(w.shape):
        raise ValueError(f'{what}: f12 {tuple(n_f12.shape)} does not match w {tuple(w.shape)}')
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= min(CONSISTENCY_MAX_K, m):
        raise ValueError(f'{what}: k={k!r} must be an integer in 1..min({CONSISTENCY_MAX_K}, M={m})')
    return s, bb, n, m


def flow_consistency(w, f12, p2, f21, k, alpha, beta, use_grid=None):
    """w [S,N,3] (the first clouds moved by the forward flows f12 [S,N,3]), p2 [B,M,3] (sample s searches p2[s % B]) and the
    reverse flows f21 [S,M,3] -> (acc [S] f64: sum_i ||r_i||^2; nn_idx [S,N,k] int32, nearest first, lowest index on ties;
    res [S,N,3]: r_i = f12_i + bhat_i, bhat_i the inverse-squared-distance interpolation of f21 over the k nearest points of
    p2; ok [S,N] uint8: ||r_i||^2 < alpha (||f12_i||^2 + ||bhat_i||^2) + beta).  F_s = acc[s] / N.  The grid form runs when p2
    has GRID_SEARCH_MIN_POINTS['laplacian'] points, the threshold of the same search (`use_grid`: see use_grid_search)."""
    s, bb, n, m = _consistency_args('flow_consistency', w, p2, f21, k, f12)
    if not (0.0 <= float(alpha) < float('inf')) or not (0.0 <= float(beta) < float('inf')):
        raise ValueError(f'flow_consistency: alpha={alpha!r} and beta={beta!r} must be finite and not negative')
    acc = torch.zeros(s, dtype=torch.float64, device=w.device)
    nn_idx = torch.empty(s, n, k, dtype=torch.int32, device=w.device)
    res = torch.empty_like(w)
    ok = torch.empty(s, n, dtype=torch.uint8, device=w.device)
    ws = _det_workspace(lib().pvraft_flow_consistency_fwd_det_workspace_bytes, s, device=w.device)
    args = (_p(w), _p(f12), _p(p2), _p(f21), s, bb, n, m, k, float(alpha), float(beta), _p(nn_idx, torch.int32), _p(res),
            _p(ok, torch.uint8), _p(acc, torch.float64))
    if use_grid_search('laplacian', m, use_grid):
        gw = _workspace(lib().pvraft_grid_index_workspace_bytes(bb, m), w.device)
        _count(lib().pvraft_flow_consistency_grid_fwd(*args, _p(gw, torch.uint8), _p(ws, torch.uint8), _stream()), 'flow_consistency_grid_fwd')
    else:
        _count(lib().pvraft_flow_consistency_fwd(*args, _p(ws, torch.uint8), _stream()), 'flow_consistency_fwd')
    return acc, nn_idx, res, ok


def flow_consistency_bwd(w, p2, f21, nn_idx, res, g, want_dp2=True):
    """Gradients of F_s = acc[s] / N (flow_consistency) with nn_idx held fixed, for the upstream gradient g [S] (on the
    device) -> (d_w [S,N,3], d_f12 [S,N,3], d_p2 [B,M,3] (the distance part; None unless want_dp2), d_f21 [S,M,3])."""
    k = int(nn_idx.shape[-1]) if nn_idx.dim() == 3 else -1
    s, bb, n, m = _consistency_args('flow_consistency_bwd', w, p2, f21, k)
    if tuple(nn_idx.shape[:2]) != (s, n) or res.shape != w.shape:
        raise ValueError(f'flow_consistency_bwd: nn_idx {tuple(nn_idx.shape)} and res {tuple(res.shape)} do not match w {tuple(w.shape)}')
    if g.shape != (s,):
        raise ValueError(f'flow_consistency_bwd: expected g [{s}], got {tuple(g.shape)}')
    d_w = torch.empty_like(w)
    d_f12 = torch.empty_like(w)
    d_p2 = torch.zeros_like(p2) if want_dp2 else None
    d_f21 = torch.zeros_like(f21)
    ws = _det_workspace(lib().pvraft_flow_consistency_bwd_det_workspace_bytes, s, bb, m, device=w.device)
    _count(lib().pvraft_flow_consistency_bwd(_p(w), _p(p2), _p(f21), _p(nn_idx, torch.int32), _p(res), _p(g), s, bb, n, m, k, _p(d_w),
                                             _p(d_f12), _p(d_p2), _p(d_f21), _p(ws, torch.uint8), _stream()), 'flow_consistency_bwd')
    return d_w, d_f12, d_p2, d_f21


PROPAGATE_MAX_K = 8   # neighbours pvraft_flow_propagate_fwd averages over at most


def flow_propagate(xyz_prev, flow_prev, xyz, k=3, want_idx=False, use_grid=None):
    """Carry a flow defined on one cloud onto another under a constant-velocity assumption: flow_prev [B,M,3] on the points
    xyz_prev [B,M,3] -> flow [B,N,3] on xyz [B,N,3], the inverse-distance-weighted mean flow of the k nearest moved points
    xyz_prev + flow_prev of every point of xyz (include/pvraft_b200.h, pvraft_flow_propagate_fwd).  want_idx: also the
    neighbours [B,N,k] int32, nearest first (exact distance ties: the lowest index).  Bitwise reproducible in any mode.  The
    grid form (the same bits) runs when xyz_prev has GRID_SEARCH_MIN_POINTS['flow_propagate'] points (`use_grid`: see use_grid_search)."""
    for name, t in (('xyz_prev', xyz_prev), ('flow_prev', flow_prev), ('xyz', xyz)):
        if not torch.is_tensor(t) or t.dim() != 3 or t.shape[-1] != 3 or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError(f'flow_propagate: expected {name} [B,n,3] with B, n >= 1, got '
                             f'{tuple(t.shape) if torch.is_tensor(t) else type(t)}')
        if t.dtype != torch.float32:
            raise ValueError(f'flow_propagate: {name} must be float32, got {t.dtype}')
    b, m = int(xyz_prev.shape[0]), int(xyz_prev.shape[1])
    if flow_prev.shape != xyz_prev.shape:
        raise ValueError(f'flow_propagate: flow_prev {tuple(flow_prev.shape)} must match xyz_prev {tuple(xyz_prev.shape)}')
    if xyz.shape[0] != b:
        raise ValueError(f'flow_propagate: xyz {tuple(xyz.shape)} and xyz_prev {tuple(xyz_prev.shape)} differ in batch size')
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= min(PROPAGATE_MAX_K, m):
        raise ValueError(f'flow_propagate: k={k!r} must be an integer in 1..min({PROPAGATE_MAX_K}, M={m})')
    for t in (xyz_prev, flow_prev, xyz):
        if not t.is_cuda:
            raise _lib.PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')
    n = int(xyz.shape[1])
    xyz_prev, flow_prev, xyz = xyz_prev.contiguous(), flow_prev.contiguous(), xyz.contiguous()
    out = torch.empty(b, n, 3, dtype=torch.float32, device=xyz.device)
    idx = torch.empty(b, n, k, dtype=torch.int32, device=xyz.device) if want_idx else None
    if use_grid_search('flow_propagate', m, use_grid):
        gw = _workspace(lib().pvraft_grid_index_workspace_bytes(b, m), xyz.device)
        _count(lib().pvraft_flow_propagate_grid_fwd(_p(xyz_prev), _p(flow_prev), _p(xyz), b, m, n, k, _p(out), _p(idx, torch.int32),
                                                    _p(gw, torch.uint8), _stream()), 'flow_propagate_grid_fwd')
        return (out, idx) if want_idx else out
    _count(lib().pvraft_flow_propagate_fwd(_p(xyz_prev), _p(flow_prev), _p(xyz), b, m, n, k, _p(out), _p(idx, torch.int32), _stream()),
           'flow_propagate_fwd')
    return (out, idx) if want_idx else out


def device_info():
    sm, smem = C.c_int(0), C.c_int(0)
    check(lib().pvraft_device_info(C.byref(sm), C.byref(smem)), 'device_info')
    return sm.value, smem.value
