"""Synthetic (H, N, C) prediction slabs for the CODA acquisition hot path.

SURVEY.md section 8(d): label-conditioned, argmax-unambiguous, generated in fixed
blocks of 65 536 points so the bytes of point n do not depend on how the N axis
is sharded.  Per block b the generator is seeded ``seed * 2**20 + b``.

  y_n        ~ Uniform{0..C-1}
  a_h        = linspace(0.55, 0.92, H)[perm(seed)]          (model accuracies)
  p_h(n)     = y_n                       w.p. a_h
             = y_n + {1,2,3} (mod C)     w.p. (1-a_h) * 0.9   ("confusion set")
             = uniform over the rest     w.p. (1-a_h) * 0.1
  kappa      ~ U(0.5, 0.99),  u ~ U(0,1)^C
  preds[h,n] = kappa * onehot(p_h(n)) + (1-kappa) * u / sum(u)      (fp32, rows sum to 1)

``dense=True`` draws the wrong class uniformly over all other classes (the
worst case for the z-sparsity of the EIG kernel).

The draw order inside a block is part of the format: labels first, then for
each group of ``H_GROUP`` models: r_correct, r_conf, r_pick, kappa, u.
"""
from __future__ import annotations

import math
import torch

BLOCK = 65536
H_GROUP = 32


def model_accuracies(H: int, seed: int) -> torch.Tensor:
    g = torch.Generator(device="cpu")
    g.manual_seed(seed * (1 << 20) + (1 << 19))
    acc = torch.linspace(0.55, 0.92, H, dtype=torch.float32)
    return acc[torch.randperm(H, generator=g)]


def _block(H, C, seed, block, device, dense, acc, out_preds, out_labels, lo, hi, want_preds=True):
    """Generate points [lo, hi) of ``block`` (block-relative) into the output views."""
    dev = torch.device(device)
    g = torch.Generator(device=dev)
    g.manual_seed(seed * (1 << 20) + block)
    y = torch.randint(0, C, (BLOCK,), generator=g, device=dev)
    if out_labels is not None:
        out_labels.copy_(y[lo:hi])
    if not want_preds:
        return
    n_conf = min(3, C - 1)
    n_rest = C - 1 - n_conf
    for h0 in range(0, H, H_GROUP):
        h1 = min(h0 + H_GROUP, H)
        hg = H_GROUP  # always draw a full group so the stream does not depend on H % H_GROUP
        r_correct = torch.rand((hg, BLOCK), generator=g, device=dev)
        r_conf = torch.rand((hg, BLOCK), generator=g, device=dev)
        r_pick = torch.rand((hg, BLOCK), generator=g, device=dev)
        kappa = torch.rand((hg, BLOCK), generator=g, device=dev) * 0.49 + 0.5
        a = torch.zeros(hg, device=dev)
        a[: h1 - h0] = acc[h0:h1].to(dev)
        correct = r_correct < a[:, None]
        if dense or n_rest <= 0:
            # wrong class uniform over the C-1 others
            off = 1 + torch.clamp((r_pick * (C - 1)).long(), max=C - 2) if C > 1 else torch.zeros_like(y)[None]
        else:
            in_conf = r_conf < 0.9
            off_conf = 1 + torch.clamp((r_pick * n_conf).long(), max=n_conf - 1)
            off_rest = 1 + n_conf + torch.clamp((r_pick * n_rest).long(), max=n_rest - 1)
            off = torch.where(in_conf, off_conf, off_rest)
        p = torch.where(correct, y[None, :], (y[None, :] + off) % C)           # (hg, BLOCK)
        for hh in range(h1 - h0):
            # u is drawn per model to bound the temporary at BLOCK*C floats
            u = torch.rand((BLOCK, C), generator=g, device=dev)
            u = u[lo:hi]
            u = u / u.sum(-1, keepdim=True)
            k = kappa[hh, lo:hi, None]
            row = (1.0 - k) * u
            row.scatter_add_(1, p[hh, lo:hi, None], k)
            out_preds[h0 + hh].copy_(row)
        # keep the stream position independent of H: burn the unused models' u draws
        for _ in range(h1 - h0, hg):
            torch.rand((BLOCK, C), generator=g, device=dev)


def synth(H: int, N: int, C: int, seed: int = 0, device="cpu", dense: bool = False,
          n_lo: int = 0, n_hi: int | None = None, want_preds: bool = True, dtype=torch.float32):
    """Return (preds[H, n_hi-n_lo, C] fp32, labels[n_hi-n_lo] int64) for the global
    point range [n_lo, n_hi) of the synthetic task (H, N, C, seed).  ``dtype`` (fp16 / bf16): the same bytes as
    ``synth(...)[0].to(dtype)``, rounded model row by model row, so the fp32 slab never exists."""
    n_hi = N if n_hi is None else n_hi
    assert 0 <= n_lo <= n_hi <= N
    dev = torch.device(device)
    n = n_hi - n_lo
    preds = torch.empty((H, n, C), dtype=dtype, device=dev) if want_preds else None
    labels = torch.empty((n,), dtype=torch.int64, device=dev)
    acc = model_accuracies(H, seed)
    b_lo, b_hi = n_lo // BLOCK, math.ceil(n_hi / BLOCK) if n_hi > 0 else 0
    for b in range(b_lo, b_hi):
        g_lo, g_hi = max(n_lo, b * BLOCK), min(n_hi, (b + 1) * BLOCK)
        if g_hi <= g_lo:
            continue
        lo, hi = g_lo - b * BLOCK, g_hi - b * BLOCK
        _block(H, C, seed, b, dev, dense, acc,
               preds[:, g_lo - n_lo:g_hi - n_lo] if want_preds else None,
               labels[g_lo - n_lo:g_hi - n_lo], lo, hi, want_preds)
    return preds, labels


def shard_range(N: int, rank: int, world: int):
    """Contiguous, balanced shard of the N axis: rank r owns [N*r//W, N*(r+1)//W)."""
    return (N * rank) // world, (N * (rank + 1)) // world


def synth_compact(H: int, N: int, C: int, K: int = 4, seed: int = 0, device="cpu", n_lo: int = 0, n_hi: int | None = None,
                  want_slab: bool = True):
    """The synthetic task directly in the compact top-K form (``CompactSlab``): same label / accuracy / confusion-set
    model as ``synth`` (labels and hard predictions are drawn the same way, block-seeded, so they do not depend on the
    sharding); the score row is kappa on the predicted class, K-1 runner-up classes that share half of the remaining
    mass, and the other half spread evenly over the C-K other classes.  Returns (ids int16 (H,n,K), probs f32 (H,n,K),
    labels int64 (n,)); ids/probs are None with ``want_slab=False``."""
    n_hi = N if n_hi is None else n_hi
    assert 0 <= n_lo <= n_hi <= N and 1 <= K < C
    dev = torch.device(device)
    n = n_hi - n_lo
    ids = torch.empty((H, n, K), dtype=torch.int16, device=dev) if want_slab else None
    probs = torch.empty((H, n, K), dtype=torch.float32, device=dev) if want_slab else None
    labels = torch.empty((n,), dtype=torch.int64, device=dev)
    acc = model_accuracies(H, seed).to(dev)
    n_conf = min(3, C - 1)
    n_rest = C - 1 - n_conf
    b_lo, b_hi = n_lo // BLOCK, math.ceil(n_hi / BLOCK) if n_hi > 0 else 0
    for b in range(b_lo, b_hi):
        g_lo, g_hi = max(n_lo, b * BLOCK), min(n_hi, (b + 1) * BLOCK)
        if g_hi <= g_lo:
            continue
        lo, hi = g_lo - b * BLOCK, g_hi - b * BLOCK
        g = torch.Generator(device=dev)
        g.manual_seed(seed * (1 << 20) + b + (1 << 18))
        y = torch.randint(0, C, (BLOCK,), generator=g, device=dev)
        labels[g_lo - n_lo:g_hi - n_lo] = y[lo:hi]
        if not want_slab:
            continue
        for h0 in range(0, H, H_GROUP):
            h1 = min(h0 + H_GROUP, H)
            hg = H_GROUP
            r_correct = torch.rand((hg, BLOCK), generator=g, device=dev)
            r_conf = torch.rand((hg, BLOCK), generator=g, device=dev)
            r_pick = torch.rand((hg, BLOCK), generator=g, device=dev)
            kappa = torch.rand((hg, BLOCK), generator=g, device=dev) * 0.49 + 0.5
            share = torch.rand((hg, BLOCK, max(1, K - 1)), generator=g, device=dev) + 0.05
            a = torch.zeros(hg, device=dev)
            a[: h1 - h0] = acc[h0:h1]
            correct = r_correct < a[:, None]
            if n_rest <= 0:
                off = 1 + torch.clamp((r_pick * (C - 1)).long(), max=C - 2)
            else:
                off_conf = 1 + torch.clamp((r_pick * n_conf).long(), max=n_conf - 1)
                off_rest = 1 + n_conf + torch.clamp((r_pick * n_rest).long(), max=n_rest - 1)
                off = torch.where(r_conf < 0.9, off_conf, off_rest)
            p = torch.where(correct, y[None, :], (y[None, :] + off) % C)[: h1 - h0, lo:hi]      # (hh, m)
            k = kappa[: h1 - h0, lo:hi]
            ids[h0:h1, g_lo - n_lo:g_hi - n_lo, 0] = p.to(torch.int16)
            probs[h0:h1, g_lo - n_lo:g_hi - n_lo, 0] = k
            if K > 1:
                sh = share[: h1 - h0, lo:hi]
                sh = sh / sh.sum(-1, keepdim=True) * (0.5 * (1.0 - k))[..., None]            # runners-up: half of the rest
                sh, _ = torch.sort(sh, dim=-1, descending=True)
                stride = max(1, (C - 1) // K)
                for j in range(1, K):
                    ids[h0:h1, g_lo - n_lo:g_hi - n_lo, j] = ((p + j * stride) % C).to(torch.int16)
                    probs[h0:h1, g_lo - n_lo:g_hi - n_lo, j] = sh[..., j - 1]
    return ids, probs, labels
