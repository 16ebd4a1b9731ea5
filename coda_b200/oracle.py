"""Label oracle (reference coda/oracle.py:1-24)."""
import ctypes as ct

import numpy as np
import torch


class Oracle:
    def __init__(self, dataset, loss_fn=None):
        self.dataset = dataset
        self.loss_fn = loss_fn
        self.device = dataset.device
        self.labels = dataset.labels
        assert self.labels is not None, "Oracle needs labels!"

    def true_losses(self, preds):
        """Mean loss of every model, (H,) (coda/oracle.py:9-21).  A ``CompactSlab``, ``HostSlab`` or ``PieceSlab``
        takes the accuracy loss only, on the pieces' devices (``sharded_true_losses``)."""
        from .datasets import CompactSlab, HostSlab, PieceSlab
        if isinstance(preds, (CompactSlab, HostSlab, PieceSlab)):
            return sharded_true_losses(preds, self.labels, self.loss_fn, self.dataset.device)
        H, N, C = preds.shape
        return self.loss_fn(preds.reshape(-1, C), self.labels.repeat(H), reduction="none").view(H, N).mean(dim=1)

    def __call__(self, idx):
        return self.labels[idx].item()


def mean_factor(H, N):
    """The fp32 factor torch's CUDA mean over the last dim of an (H, N) fp32 tensor multiplies its sum by
    (ReduceMomentKernel.cu: ``float(num_output_elements) / numel``, MeanOps::project is ``a * factor``)."""
    return np.float32(H) / np.float32(H * N)


def sharded_true_losses(slab, labels, loss_fn, device):
    """``Oracle.true_losses`` of a slab in pieces (``datasets.pieces_of``) with the accuracy loss: one
    ``coda_b200_true_loss_counts`` launch per device piece, each on its device and a stream of its own, all in flight
    together.  The per-model wrong counts are exact integers below 2^24, so they equal torch's fp32 sums; the result
    carries the bits of ``true_losses`` on the same slab held as one tensor, on ``device``.

    A ``CompactSlab`` (one piece) or ``ShardedCompactSlab`` counts the items whose ``ids[0]`` -- the hard prediction
    every selector sees -- is the label (``coda_b200_true_loss_counts_compact``).  For a slab compacted from a dense one
    (``CompactSlab.from_dense``, ``load_compact``) ``ids[0]`` is the dense arg-max, so the result has the bits of
    ``true_losses`` on the dense slab.  It can differ from ``true_losses(slab.densify())`` only in the rows counted in
    ``compaction["flat_rows"]``, where the uniform remainder reaches ``probs[0]``.

    A ``HostSlab`` piece is counted chunk by chunk as it streams through its device (``HostSlab.walk``), after the
    device pieces before it are in flight and before the pieces after it start."""
    from . import _native as nat
    from .datasets import CompactSlab, model_stride, pieces_of, walk
    name = type(slab).__name__
    try:
        from coda.options import accuracy_loss                # what LOSS_FNS["acc"] resolves to
    except ImportError:
        accuracy_loss = None
    if accuracy_loss is None or loss_fn is not accuracy_loss:
        raise NotImplementedError(f"Oracle.true_losses on a {name} takes the accuracy loss only "
                                  "(coda.options.accuracy_loss, LOSS_FNS['acc'])")
    if labels.dim() != 1:
        raise NotImplementedError(f"Oracle.true_losses on a {name} takes 1-D class labels")
    H, N, C = (int(s) for s in slab.shape)
    if N >= 1 << 24:
        raise NotImplementedError(f"Oracle.true_losses on a {name}: N = {N} >= 2^24, where fp32 sums of the "
                                  f"per-item losses stop being exact counts")
    if not slab.is_cuda:
        raise NotImplementedError(f"coda_b200: the pieces of a {name} must be CUDA tensors; there is no CPU path")
    lib = nat.load()
    labels = labels.to(torch.int64)
    parts = []
    for piece, off in pieces_of(slab):
        dev = piece.device
        n = int(piece.shape[1])
        with torch.cuda.device(dev):
            st = torch.cuda.Stream(device=dev)
            st.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(st):
                lab = labels[off:off + n].to(dev, non_blocking=False)
                if isinstance(piece, CompactSlab):
                    cnt = torch.empty(H, dtype=torch.int64, device=dev)
                    nat.check(lib.coda_b200_true_loss_counts_compact(
                        ct.c_void_p(piece.ids.data_ptr()), model_stride(piece.ids), H, n, piece.K,
                        ct.c_void_p(lab.data_ptr()), ct.c_void_p(cnt.data_ptr()), ct.c_void_p(st.cuda_stream)),
                        "true_loss_counts_compact")
                    parts.append((cnt, st))
                else:
                    def body(n0, n1, v):
                        cnt = torch.empty(H, dtype=torch.int64, device=dev)
                        nat.check(lib.coda_b200_true_loss_counts(ct.c_void_p(v.data_ptr()), nat.slab_format(v.dtype),
                                                                 model_stride(v), H, n1 - n0, C,
                                                                 ct.c_void_p(lab[n0:].data_ptr()),
                                                                 ct.c_void_p(cnt.data_ptr()), ct.c_void_p(st.cuda_stream)),
                                  "true_loss_counts")
                        parts.append((cnt, st))
                    walk(piece, body)          # a host piece returns when its chunks are counted
                lab.record_stream(st)
    correct = torch.zeros(H, dtype=torch.int64, device=device)
    for cnt, st in parts:
        st.synchronize()
        correct += cnt.to(device)
    wrong = (N - correct).to(torch.float32)                 # sum of the 0/1 losses, exact
    return wrong * torch.tensor(mean_factor(H, N), device=device)
