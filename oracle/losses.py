"""Oracle restatement of the reference losses (TEST INFRASTRUCTURE).

  dice_loss      training/losses.py:18-58  (adaptive Tversky; alpha stays in the autograd graph, :38-41)
  cross_entropy  nn.CrossEntropyLoss(weight) as called at train_ddp.py:93,189-191
  total_loss     sum over heads with aux weights, train_ddp.py:186-191
"""
import torch
import torch.nn.functional as F

SMOOTH = 1e-5


def dice_terms(preds, targets):
    """Per-class terms of dice_loss: (alpha before the clamp, alpha, dice), each [C]."""
    P = F.softmax(preds if preds.dtype == torch.float64 else preds.float(), dim=1)
    M = torch.zeros_like(P).scatter_(1, targets, 1.0)
    dims = [0] + list(range(2, P.dim()))           # batch and space jointly (losses.py:38-44)
    TP = (P * M).sum(dims)
    FP = (P * (1 - M)).sum(dims)
    FN = ((1 - P) * M).sum(dims)
    alpha_raw = FP / (FP + FN + SMOOTH)
    alpha = torch.clamp(alpha_raw, min=0.2, max=0.8)
    beta = 1 - alpha
    dice = TP / (TP + alpha * FP + beta * FN + SMOOTH)
    return alpha_raw, alpha, dice


def dice_loss(preds, targets):
    """preds [B,C,...] float, targets [B,1,...] int64."""
    C = preds.shape[1]
    dice = dice_terms(preds, targets)[2]
    return (1 - dice).sum() / C


def cross_entropy(preds, targets, weight=None):
    x = preds if preds.dtype == torch.float64 else preds.float()
    return F.cross_entropy(x, targets.squeeze(1), weight=None if weight is None else weight.to(x.dtype))


def total_loss(result, label, weight=None, aux_weight=None):
    if isinstance(result, (list, tuple)):
        return sum(aux_weight[j] * (cross_entropy(r, label, weight) + dice_loss(r, label)) for j, r in enumerate(result))
    return cross_entropy(result, label, weight) + dice_loss(result, label)
