"""fp64 torch model of link prediction (Distributed_Sparse::linkLoss, include/hnh/training.hpp) -- TEST INFRASTRUCTURE.

For the stored entries (rows[i], cols[i]) of a target matrix T with targets y[i]:
    s    = (H_A[rows] * H_B[cols]).sum(1)
    loss = F.binary_cross_entropy_with_logits(s, y, reduction="mean")     (0 and a zero gradient without entries)
    correct = #[(s > 0) == (y > 0.5)]
and the gradients by autograd.  Link training is tests/training_oracle.py's step (torch.optim.AdamW(foreach=False),
clip_grad_norm_) with this loss on the output of the same forward builders: train_gt / train_gat are run with their
loss step swapped for link_train_step below, so the models are exactly those of node classification.  fp64 on the CPU;
nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import math
from unittest import mock

import numpy as np
import torch
import torch.nn.functional as F

from tests import training_oracle as tro


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def bce_terms(s, y):
    """The stable per-entry loss max(s, 0) - s y + log1p(exp(-|s|)) (torch tensors)."""
    return torch.clamp(s, min=0) - s * y + torch.log1p(torch.exp(-s.abs()))


def link_loss(H_A, H_B, rows, cols, y, same=False):
    """(loss, correct, count, scores, dH_A, dH_B) as numpy / Python numbers.  same=True: H_A is H_B, one leaf, and
    dH_A = dH_B is its whole gradient."""
    rows, cols = torch.as_tensor(np.asarray(rows, np.int64)), torch.as_tensor(np.asarray(cols, np.int64))
    yt = _t(y)
    a = _t(H_A).clone().requires_grad_()
    b = a if same else _t(H_B).clone().requires_grad_()
    s = (a[rows] * b[cols]).sum(1)
    loss = F.binary_cross_entropy_with_logits(s, yt, reduction="mean") if len(yt) else (a * 0).sum() + (b * 0).sum()
    loss.backward()
    correct = int(((s.detach() > 0) == (yt > 0.5)).sum())
    ga = a.grad.numpy().copy()
    gb = ga if same else b.grad.numpy().copy()
    return float(loss.detach()), correct, len(yt), s.detach().numpy(), ga, gb


def link_train_step(pairs):
    """The loss step of tests/training_oracle.train for link prediction: `labels` is (rows, cols, y)."""
    rows, cols, y = pairs

    def train(forward, params, _labels, steps, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=None,
              lrs=None):
        opt = torch.optim.AdamW(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, foreach=False)
        r, c, yt = torch.as_tensor(np.asarray(rows, np.int64)), torch.as_tensor(np.asarray(cols, np.int64)), _t(y)
        out = []
        for t in range(steps):
            if lrs is not None:
                opt.param_groups[0]["lr"] = lrs[t]
            opt.zero_grad()
            H = forward(t)
            s = (H[r] * H[c]).sum(1)
            loss = F.binary_cross_entropy_with_logits(s, yt, reduction="mean") if len(yt) else (H * 0).sum()
            loss.backward()
            for p in params:
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
            norm = torch.nn.utils.clip_grad_norm_(params, max_grad_norm if max_grad_norm else math.inf)
            correct = int(((s.detach() > 0) == (yt > 0.5)).sum())
            out.append((float(loss.detach()), correct, len(yt), float(norm)))
            opt.step()
        return out

    return train


def train_gt(rows, cols, N, layers, params, X, pairs, steps, **kw):
    """tests/training_oracle.train_gt with the link loss over pairs = (T rows, T cols, targets)."""
    with mock.patch.object(tro, "train", link_train_step(pairs)):
        return tro.train_gt(rows, cols, N, layers, params, X, None, steps, **kw)


def train_gat(kind, rows, cols, N, layers, weights, a1, a2, X, pairs, steps, **kw):
    """tests/training_oracle.train_gat with the link loss over pairs = (T rows, T cols, targets)."""
    with mock.patch.object(tro, "train", link_train_step(pairs)):
        return tro.train_gat(kind, rows, cols, N, layers, weights, a1, a2, X, None, steps, **kw)


def auc(scores, y):
    """The area under the ROC curve of scores against binary targets y (ties count one half)."""
    scores, y = np.asarray(scores), np.asarray(y) > 0.5
    pos, neg = scores[y], scores[~y]
    if not len(pos) or not len(neg):
        return math.nan
    order = np.argsort(np.concatenate([pos, neg]), kind="mergesort")
    ranks = np.empty(len(order))
    allv = np.concatenate([pos, neg])[order]
    # average ranks over ties
    i = 0
    while i < len(allv):
        j = i
        while j + 1 < len(allv) and allv[j + 1] == allv[i]:
            j += 1
        ranks[order[i:j + 1]] = (i + j) / 2 + 1
        i = j + 1
    return float((ranks[:len(pos)].sum() - len(pos) * (len(pos) + 1) / 2) / (len(pos) * len(neg)))
