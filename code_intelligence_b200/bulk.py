"""Multi-GPU bulk per-repo encode (BASELINE.json config 4; SURVEY.md section 8e).

Issues are independent (the encoder state is reset per call, inference.py:56), so the path shards with no data-path
collective: global argsort by length (py/code_intelligence/inference.py:192-194), sorted position j goes to rank
``j mod G`` (every rank sees the same length distribution), each rank encodes its shard with its own weight replica,
and exactly ONE exchange step follows -- an all-gather of the (ceil(N/G), 2400) float32 outputs (NCCL over NVLink on
GPUs; gloo in the CPU tests) -- before the inverse permutation restores input order (inference.py:226).
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np


def _to_numpy(t) -> np.ndarray:
    """Device tensor -> np.ndarray through page-locked host memory.  ``tensor.cpu()`` lands in fresh pageable pages (first
    touch faults + the driver's bounce buffers: ~4 GB/s measured for the (N, 2400) result, 12.6 ms per 49 MB); torch's
    caching pinned allocator hands the same block back call after call, and the returned array owns it (the block
    returns to that cache when the array is dropped)."""
    import torch
    if not t.is_cuda:
        return t.numpy()
    if t.numel() * t.element_size() > (2 << 30):
        # a FRESH page-locked block of this size costs more than it saves (measured for the 9.6 GB result of a
        # 1 M-issue encode: cudaHostAlloc 4.97 s + copy 0.17 s, against 2.77 s for the pageable copy); only repeated
        # calls of the same size would get the cached block back
        return t.cpu().numpy()
    try:
        host = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    except RuntimeError:
        return t.cpu().numpy()
    host.copy_(t)
    return host.numpy()


def encode_sorted_batches(docs: List[np.ndarray], encode_padded: Callable, pad_idx: int, out_dim: int, bs: int = 100,
                          max_bs: int = 256, min_batches_rule: bool = True, coalesce: bool = False) -> np.ndarray:
    """The single-device bulk loop of ``df_to_embedding`` from the numericalised docs on
    (py/code_intelligence/inference.py:171-229): ``bs = min(bs, N//20 + 1)`` (at least 20 batches so that length
    sorting pays), argsort by length, batches of ``bs`` consecutive sorted docs right-padded to the batch's own max
    with ``pad_idx`` (pad_sequence, :207), ``encode_padded(ids[B,T], lengths[B]) -> (B, out_dim)``, on
    ``RuntimeError`` (CUDA OOM, :214-223) halve ``bs`` and retry the same position -- re-raised as ``Exception`` at
    bs == 1 -- and finally unsort with argsort(argsort) (:226).

    ``coalesce=True``: consecutive sorted batches are merged into device calls of ``max_bs`` rows.  On the GPU path a
    row's result does not depend on its batch mates or on the padded length (bit-exact, tests/test_gpu_parity.py), so
    ``bs`` -- a memory knob of the reference, default 100 -- only decides how many rows ride one launch; merging keeps
    the results and lets a caller with the reference's default arguments reach full 1280-row launches."""
    n = len(docs)
    if n == 0:
        return np.empty((0, out_dim), dtype=np.float32)
    if min_batches_rule:
        bs = min(bs, (n // 20) + 1)
    bs = max(1, min(bs, max_bs))
    if coalesce:
        bs = max_bs
    length_arr = np.array([len(d) for d in docs])
    if (length_arr < 1).any():
        raise ValueError("empty token sequence")
    len_mask = length_arr.argsort(kind="stable")
    len_mask_reversed = len_mask.argsort()
    ordered_lengths = length_arr[len_mask]
    pooled = np.empty((n, out_dim), dtype=np.float32)
    i = 0
    while i < n:
        try:
            idx = len_mask[i:i + bs]
            T = int(ordered_lengths[i + len(idx) - 1])
            bp = np.full((len(idx), T), pad_idx, dtype=np.int64)
            for r, j in enumerate(idx):
                bp[r, :length_arr[j]] = docs[j]
            pooled[i:i + len(idx)] = encode_padded(bp, ordered_lengths[i:i + len(idx)].astype(np.int32))
            i += bs
        except RuntimeError as e:
            if bs == 1:
                raise Exception(e)
            bs = max(1, min(bs, n - i) // 2)     # halve what was actually attempted (the tail may be shorter than bs)
    assert pooled.shape[0] == length_arr.shape[0]
    return pooled[len_mask_reversed, :]


def encode_sorted_batches_device(docs: List[np.ndarray], enc, bs: int = 100, min_batches_rule: bool = True,
                                 coalesce: bool = True, to_host: bool = True):
    """The same bulk loop as ``encode_sorted_batches`` driven as a pipeline on the GPU (``enc``: an ``IssueEncoder``):
    the padded batch k+1 is packed into pinned host memory and copied to the device on a side stream while the kernels
    of batch k run (two staging slots, events instead of host synchronisation), the pooled rows of every batch land in
    one device tensor, and the un-sort (argsort(argsort), py/code_intelligence/inference.py:226) is one device gather.
    ``IE_ERR_OOM`` still surfaces as ``RuntimeError`` at the call that needed the memory (workspace is allocated before
    anything is launched), so the reference's halving loop (:214-223) keeps its meaning.
    Returns np.ndarray (N, D) float32 in input order, or the device tensor with ``to_host=False``."""
    import torch
    n = len(docs)
    D = enc.out_dim
    dev = torch.device("cuda", enc.device)
    if n == 0:
        return np.empty((0, D), dtype=np.float32) if to_host else torch.empty((0, D), dtype=torch.float32, device=dev)
    max_bs = enc.max_batch
    if min_batches_rule:
        bs = min(bs, (n // 20) + 1)
    bs = max(1, min(bs, max_bs))
    if coalesce:
        bs = max_bs
    length_arr = np.array([len(d) for d in docs])
    if (length_arr < 1).any():
        raise ValueError("empty token sequence")
    len_mask = length_arr.argsort(kind="stable")
    ordered_lengths = length_arr[len_mask]
    with torch.cuda.device(dev):
        out = torch.empty((n, D), dtype=torch.float32, device=dev)      # sorted order
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)

        class Slot:
            def __init__(self):
                self.ids_pin = self.len_pin = self.ids_dev = self.len_dev = None
                self.h2d_done, self.compute_done = torch.cuda.Event(), torch.cuda.Event()
                self.used = False

            def reserve(self, tokens, rows):
                if self.ids_pin is None or self.ids_pin.numel() < tokens:
                    self.ids_pin = torch.empty(tokens, dtype=torch.int64).pin_memory()
                    self.ids_dev = torch.empty(tokens, dtype=torch.int64, device=dev)
                if self.len_pin is None or self.len_pin.numel() < rows:
                    self.len_pin = torch.empty(rows, dtype=torch.int32).pin_memory()
                    self.len_dev = torch.empty(rows, dtype=torch.int32, device=dev)

        slots = [Slot(), Slot()]
        i, k = 0, 0
        while i < n:
            nb = min(bs, n - i)
            idx = len_mask[i:i + nb]
            T = int(ordered_lengths[i + nb - 1])
            st = slots[k & 1]
            if st.used:
                st.compute_done.synchronize()       # the slot's device buffers (and so its staging) are free again
            st.reserve(nb * T, nb)
            bp = st.ids_pin[:nb * T].view(nb, T).numpy()
            lens = ordered_lengths[i:i + nb]
            if int(lens[0]) == T:                    # fixed-length batch: one vectorised copy
                bp[:] = np.stack([docs[j] for j in idx])
            else:
                bp.fill(enc.pad_idx)
                for r, j in enumerate(idx):
                    bp[r, :length_arr[j]] = docs[j]
            st.len_pin[:nb].numpy()[:] = lens
            with torch.cuda.stream(side):
                st.ids_dev[:nb * T].copy_(st.ids_pin[:nb * T], non_blocking=True)
                st.len_dev[:nb].copy_(st.len_pin[:nb], non_blocking=True)
                st.h2d_done.record(side)
            cur.wait_event(st.h2d_done)
            try:
                enc.encode_ids_device(st.ids_dev[:nb * T].view(nb, T), st.len_dev[:nb], out[i:i + nb], cur)
            except RuntimeError as e:
                if bs == 1:
                    raise Exception(e)
                bs = max(1, nb // 2)                 # halve what was actually attempted and retry the same position
                st.h2d_done.synchronize()            # the staging buffer is about to be re-packed
                continue
            st.compute_done.record(cur)
            st.used = True
            i += nb
            k += 1
        enc.check_errors()                           # token ids out of range etc. (device-pointer calls are asynchronous)
        inv = torch.as_tensor(len_mask.argsort(), device=dev)
        res = out.index_select(0, inv)
    return _to_numpy(res) if to_host else res


def shard_plan(lengths: np.ndarray, world: int):
    """-> (order, shards): order = stable argsort by length; shards[r] = input indices of rank r (sorted order)."""
    order = np.asarray(lengths).argsort(kind="stable")
    return order, [order[r::world] for r in range(world)]


def gather_rows(local, n_total: int, world: int, rank: int, group=None):
    """local: torch tensor (n_r, D) of this rank's rows in sorted-position order r, r+G, r+2G, ...
    Returns (n_total, D) in sorted order on every rank.  One all_gather."""
    import torch
    import torch.distributed as dist
    per = (n_total + world - 1) // world
    D = local.shape[1]
    buf = torch.zeros((per, D), dtype=local.dtype, device=local.device)
    buf[:local.shape[0]] = local
    if world == 1:
        allr = buf[None]
    else:
        allr = torch.empty((world, per, D), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(allr.view(world * per, D), buf, group=group)
    # sorted position j = k*world + r  <-  allr[r, k]
    return allr.transpose(0, 1).reshape(per * world, D)[:n_total]


def encode_bulk_distributed(docs: List[np.ndarray], encode_local: Callable[[List[np.ndarray]], "np.ndarray"],
                            device: Optional[str] = None, group=None, to_host=True):
    """Every rank passes the same ``docs`` (the reference's per-repo list) and gets the full (N, D) float32 array in
    input order.  ``encode_local(list_of_id_arrays) -> (n, D)`` is the per-rank encoder; it may return a numpy array
    (CPU / gloo tests) or a torch tensor that already lives on the GPU -- e.g.
    ``lambda d: bulk.encode_sorted_batches_device(d, enc, min_batches_rule=False, to_host=False)`` -- in which case
    nothing bounces through the host: the all-gather (NCCL over NVLink) and the inverse permutation run on the device.
    ``to_host``: True -> numpy on every rank; "rank0" -> numpy on rank 0, the device tensor elsewhere; False -> tensor."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n = len(docs)
    lengths = np.array([len(d) for d in docs])
    order, shards = shard_plan(lengths, world)
    mine = [docs[i] for i in shards[rank]]
    local = encode_local(mine) if len(mine) else None
    if local is None:
        lt = torch.zeros((0, 0), dtype=torch.float32)
    elif isinstance(local, torch.Tensor):
        lt = local.to(torch.float32)
    else:
        lt = torch.as_tensor(np.ascontiguousarray(local, dtype=np.float32))
    if device is not None and str(lt.device) != str(device):
        lt = lt.to(device)
    # every rank must agree on D even when its shard is empty
    d_t = torch.tensor([lt.shape[1] if lt.shape[0] else 0], dtype=torch.int64, device=lt.device)
    if world > 1:
        dist.all_reduce(d_t, op=dist.ReduceOp.MAX, group=group)
    D = int(d_t.item())
    if lt.shape[0] == 0:
        lt = torch.zeros((0, D), dtype=torch.float32, device=lt.device)
    sorted_rows = gather_rows(lt.contiguous(), n, world, rank, group)
    inv = torch.as_tensor(order.argsort(), device=sorted_rows.device)
    res = sorted_rows.index_select(0, inv)
    if to_host == "rank0":        # the reference's driver is one process: only rank 0 needs the array on the host
        return _to_numpy(res) if rank == 0 else res
    return _to_numpy(res) if to_host else res
