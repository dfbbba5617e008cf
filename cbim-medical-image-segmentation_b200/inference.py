"""Evaluation-side consumers of ``net(x)`` behind the reference's own function names (SURVEY.md §8f.2):
  inference_whole_image / inference_sliding_window / get_inference   inference/inference3d.py:8-92, inference/utils.py:1-40
  inference_whole_image_2d / inference_sliding_window_2d            inference/inference2d.py (D = 1 on the same kernels)
  calculate_dice / calculate_dice_split                               metric/utils.py:33-82
  calculate_distance                                                  metric/utils.py:8-28
Same signatures and return values (probabilities fp32 [B,classes,D,H,W]; (dice, intersection, summ) tensors); the
window schedule (half-window stride, last window snapped to the border, utils.split_idx) is the reference's.  On the
device the per-window softmax + accumulate + count is ONE kernel, the final division (and an optional argmax label
map) another, and the Dice metric is a single pass over the two label maps — the [N,C] one-hot masks never exist.
The surface distances (ASD, percentile HD) run on the device too (csrc/surface.cu, DESIGN.md §3.10)."""
import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from .ops import _dt, _need_cuda, _stream, on_device
from .surface import surface_area_table


def split_idx(half_win, size, i):
    """inference/utils.py:27-40."""
    start = half_win * i
    end = start + half_win * 2
    if end > size:
        start, end = size - half_win * 2, size
    return start, end


def _softmax_accumulate(logits, prob, counter, region):
    """prob[region] += softmax(logits, 1); counter[region] += 1.  logits: [B,C,d,h,w]-shaped view, any strides."""
    B, C = logits.shape[0], logits.shape[1]
    d0, h0, w0, wd, wh, ww = region
    if logits.dtype not in (torch.float16, torch.float32):
        logits = logits.float()
    cl = logits.permute(0, 2, 3, 4, 1)
    if cl.is_contiguous():                       # channels-last view handed out by the b200seg models
        sb, sv, sc = cl.stride(0), C, 1
    else:
        logits = logits.contiguous()
        sb, sv, sc = logits.stride(0), 1, logits.stride(1)
    D, H, W = prob.shape[2:]
    _lib.call("b200seg_softmax_accumulate", logits.data_ptr(), _dt(logits), sb, sv, sc, prob.data_ptr(), counter.data_ptr(),
              B, C, wd, wh, ww, D, H, W, d0, h0, w0, _stream())


def inference_whole_image(net, img, args=None):
    """inference/inference3d.py:8-25."""
    net.eval()
    with torch.no_grad():
        pred = net(img)
        if isinstance(pred, (tuple, list)):
            pred = pred[0]
    _need_cuda(pred)
    with on_device(pred):
        B, C = pred.shape[:2]
        prob = torch.zeros(B, C, *pred.shape[2:], dtype=torch.float32, device=pred.device)
        counter = torch.zeros(B, 1, *pred.shape[2:], dtype=torch.float32, device=pred.device)
        _softmax_accumulate(pred, prob, counter, (0, 0, 0, *pred.shape[2:]))
    return prob


def inference_sliding_window(net, img, args, return_label=False):
    """inference/inference3d.py:28-92.  return_label=True additionally returns the uint8 argmax map produced by the
    normalisation kernel (validation_ddp's `torch.max(pred, 1)`, training/validation.py:120-135, without another pass)."""
    net.eval()
    _need_cuda(img)
    B, C, D, H, W = img.shape
    win_d, win_h, win_w = args.window_size
    flag = False
    if D < win_d or H < win_h or W < win_w:
        flag = True
        img = F.pad(img, (0, max(0, win_w - W), 0, max(0, win_h - H), 0, max(0, win_d - D)))
        origin = (D, H, W)
        B, C, D, H, W = img.shape
    hd, hh, hw = win_d // 2, win_h // 2, win_w // 2
    with on_device(img):
        prob = torch.zeros(B, args.classes, D, H, W, dtype=torch.float32, device=img.device)
        counter = torch.zeros(B, 1, D, H, W, dtype=torch.float32, device=img.device)
        with torch.no_grad():
            for i in range(D // hd):
                for j in range(H // hh):
                    for k in range(W // hw):
                        d0, d1 = split_idx(hd, D, i)
                        h0, h1 = split_idx(hh, H, j)
                        w0, w1 = split_idx(hw, W, k)
                        pred = net(img[:, :, d0:d1, h0:h1, w0:w1])
                        if isinstance(pred, (tuple, list)):
                            pred = pred[0]
                        _softmax_accumulate(pred, prob, counter, (d0, h0, w0, d1 - d0, h1 - h0, w1 - w0))
        label = torch.empty(B, D, H, W, dtype=torch.uint8, device=img.device) if return_label else None
        _lib.call("b200seg_normalize_argmax", prob.data_ptr(), counter.data_ptr(), None if label is None else label.data_ptr(),
                  B, args.classes, D * H * W, _stream())
    if flag:
        prob = prob[:, :, :origin[0], :origin[1], :origin[2]]
        if label is not None:
            label = label[:, :origin[0], :origin[1], :origin[2]]
    return (prob, label) if return_label else prob


def _logits5(pred):
    """[B,C,H,W] logits (any strides) as the [B,C,1,H,W] view the accumulation kernel takes."""
    if isinstance(pred, (tuple, list)):
        pred = pred[0]
    return pred.unsqueeze(2)


def inference_whole_image_2d(net, img, args=None):
    """inference/inference2d.py inference_whole_image: img [B,C,H,W] (a slice stack) -> softmax [B,classes,H,W]."""
    net.eval()
    with torch.no_grad():
        pred = _logits5(net(img))
    _need_cuda(pred)
    with on_device(pred):
        B, C, _, H, W = pred.shape
        prob = torch.zeros(B, C, 1, H, W, dtype=torch.float32, device=pred.device)
        counter = torch.zeros(B, 1, 1, H, W, dtype=torch.float32, device=pred.device)
        _softmax_accumulate(pred, prob, counter, (0, 0, 0, 1, H, W))
    return prob[:, :, 0]


def inference_sliding_window_2d(net, img, args):
    """inference/inference2d.py inference_sliding_window: half-window stride, last window snapped to the border
    (no padding: the image must be at least one window), softmax averaged over the windows; [B,classes,H,W]."""
    net.eval()
    _need_cuda(img)
    B, C, H, W = img.shape
    win_h, win_w = args.window_size
    hh, hw = win_h // 2, win_w // 2
    with on_device(img):
        prob = torch.zeros(B, args.classes, 1, H, W, dtype=torch.float32, device=img.device)
        counter = torch.zeros(B, 1, 1, H, W, dtype=torch.float32, device=img.device)
        with torch.no_grad():
            for i in range(H // hh):
                for j in range(W // hw):
                    h0, h1 = split_idx(hh, H, i)
                    w0, w1 = split_idx(hw, W, j)
                    pred = _logits5(net(img[:, :, h0:h1, w0:w1]))
                    _softmax_accumulate(pred, prob, counter, (0, h0, w0, 1, h1 - h0, w1 - w0))
        _lib.call("b200seg_normalize_argmax", prob.data_ptr(), counter.data_ptr(), None, B, args.classes, H * W, _stream())
    return prob[:, :, 0]


def get_inference(args):
    """inference/utils.py:1-23."""
    if args.dimension == '3d':
        return inference_sliding_window if args.sliding_window else inference_whole_image
    if args.dimension == '2d':
        return inference_sliding_window_2d if args.sliding_window else inference_whole_image_2d
    raise ValueError('Error in image dimension')


def calculate_dice(pred, target, C):
    """metric/utils.py:62-82: pred / target label tensors [N,1] (or any shape with N elements); returns
    (dice [C], intersection [C], summ [C]) float32 like the reference (summ includes its +1e-5)."""
    _need_cuda(pred)
    p = pred.reshape(-1)
    t = target.reshape(-1)
    if p.dtype not in (torch.uint8, torch.int64):
        p = p.long()
    if t.dtype not in (torch.uint8, torch.int64):
        t = t.long()
    p, t = p.contiguous(), t.contiguous()
    with on_device(p):
        out = torch.zeros(C, 2, dtype=torch.int64, device=p.device)
        _lib.call("b200seg_dice_metric", p.data_ptr(), p.element_size(), t.data_ptr(), t.element_size(), p.numel(), C,
                  out.data_ptr(), _stream())
    intersection = out[:, 0].to(torch.float32)
    summ = out[:, 1].to(torch.float32) + 1e-5
    return 2 * intersection / summ, intersection, summ


def calculate_dice_split(pred, target, C, block_size=64 * 64 * 64):
    """metric/utils.py:33-55: the reference splits only to bound the memory of its one-hot masks; the device kernel has
    none, so this is one pass with the reference's final formula."""
    _, inter, summ = calculate_dice(pred, target, C)
    summ = summ - 1e-5
    return 2 * inter / (summ + 1e-5), inter, summ


def calculate_distance(label_pred, label_true, spacing, C, percentage=95):
    """metric/utils.py:8-28: label maps [D,H,W] (CUDA, any integer dtype; uint8 / int64 are read in place), spacing
    (tensor, ndarray or sequence of 3) -> (ASD_list, HD_list), numpy float64 [C-1]: per class 1..C-1 the mean of the
    two directed average surface distances and the larger of the two directed `percentage` percentile distances.
    A class missing from one or both maps gives nan / inf, as the reference (validation_ddp clips them itself)."""
    if label_pred.dim() != 3 or label_true.dim() != 3:
        raise ValueError("calculate_distance takes 3-D label maps, got %d-D and %d-D" % (label_pred.dim(), label_true.dim()))
    if label_pred.shape != label_true.shape:
        raise ValueError("label maps differ in shape: %s vs %s" % (tuple(label_pred.shape), tuple(label_true.shape)))
    if C > 256:
        raise _lib.B200SegError("calculate_distance supports at most 256 classes, got %d" % C)
    _need_cuda(label_pred)
    _need_cuda(label_true)
    if isinstance(spacing, torch.Tensor):
        spacing = spacing.detach().cpu().double().tolist()
    spacing = [float(s) for s in np.asarray(spacing, dtype=np.float64).reshape(-1)]
    table = surface_area_table(spacing)
    maps = []
    for t in (label_pred, label_true):
        if t.dtype not in (torch.uint8, torch.int64):
            t = t.long()
        maps.append(t.contiguous())
    p, t = maps
    D, H, W = p.shape
    if C < 2:
        return np.zeros(0), np.zeros(0)
    with on_device(p):
        table_d = torch.from_numpy(table).to(p.device)
        out = torch.empty(2, C - 1, dtype=torch.float64, device=p.device)
        ws_bytes = _lib.load().b200seg_surface_distance_workspace(D, H, W, C)
        if ws_bytes == 0:
            raise _lib.B200SegError("calculate_distance: unsupported volume %dx%dx%d" % (D, H, W))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=p.device)
        _lib.call("b200seg_surface_distance", p.data_ptr(), p.element_size(), t.data_ptr(), t.element_size(), D, H, W, C,
                  spacing[0], spacing[1], spacing[2], float(percentage), table_d.data_ptr(), out[0].data_ptr(),
                  out[1].data_ptr(), ws.data_ptr(), ws_bytes, _stream())
        res = out.cpu().numpy()
    return res[0].copy(), res[1].copy()
