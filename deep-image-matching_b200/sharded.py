"""Multi-GPU driver of the hot path (SURVEY 8e): one process per GPU (torch.distributed; nccl on GPUs, gloo in the CPU tests).

Independent-pair workloads (bench.py default): pairs are dealt to ranks, no data-path collective, one gather of the match
tables to rank 0.  Image-set workloads (exhaustive / sequential pair lists over n images - ImageMatcher.extract_features +
match_pairs, image_matching.py:413-494, is the serial loop this replaces) run in two phases:
  1. image i is extracted on rank ``i % G`` into that rank's region of the device feature store (``shard_images``,
     ``store_slot``);
  2. ONE ``all_gather`` of the float16 feature blocks (NCCL over NVLink; ~1.07 MB per SuperPoint image) gives every rank all
     features (``all_gather_blocks``), then the pair list is dealt by longest-processing-time (``shard_pairs``) and each rank
     matches its pairs (LightGlue or SuperGlue) out of its own HBM; the variable-length match tables are gathered to rank 0
     (``gather_match_tables``)."""
from __future__ import annotations

import numpy as np


def shard_pairs(n_pairs: int, world: int, rank: int, costs=None) -> list:
    """Indices of the pairs rank `rank` processes.  Round-robin by default (pairs_from_bruteforce order,
    pairs_generator.py:37-38); with per-pair costs (e.g. N0*N1) a longest-processing-time deal balances the
    early-exit variance.  Deterministic on every rank."""
    if costs is None:
        return list(range(rank, n_pairs, world))
    order = sorted(range(n_pairs), key=lambda i: (-float(costs[i]), i))
    load = [0.0] * world
    mine = []
    for i in order:
        r = min(range(world), key=lambda k: (load[k], k))
        load[r] += float(costs[i])
        if r == rank:
            mine.append(i)
    return sorted(mine)


def shard_images(n_images: int, world: int, rank: int) -> list:
    """Images rank `rank` extracts: i % world == rank (tiles of one image stay on one rank)."""
    return list(range(rank, n_images, world))


def images_per_rank(n_images: int, world: int) -> int:
    return (n_images + world - 1) // world


def store_slot(image: int, n_images: int, world: int) -> int:
    """Slot of image `image` in the device feature store: rank-major, so that each rank's extractions are one contiguous run of
    blocks and the exchange is a single all_gather of equal-sized regions."""
    return (image % world) * images_per_rank(n_images, world) + image // world


def all_gather_blocks(store_tensor, n_images: int, dist=None):
    """store_tensor: uint8 tensor viewing the whole store, shape (world * images_per_rank, slot_bytes); rank r has filled rows
    [r * ipr, (r + 1) * ipr).  After the call every rank holds every block.  Returns the bytes this rank received."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return 0
    world, rank = dist.get_world_size(), dist.get_rank()
    ipr = images_per_rank(n_images, world)
    assert store_tensor.shape[0] == world * ipr, (store_tensor.shape, world, ipr)
    mine = store_tensor[rank * ipr:(rank + 1) * ipr].clone()  # send buffer (the receive buffer is the store itself)
    dist.all_gather_into_tensor(store_tensor.view(-1), mine.view(-1))
    return (world - 1) * mine.numel()


def gather_match_tables(local_ids, local_matches, n_pairs: int, dist=None, device=None):
    """Gather {pair id -> int64 (S,2)} from all ranks to rank 0 (counts all_gather + padded all_gather).
    Returns the full list on rank 0 (None elsewhere)."""
    import torch

    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        out = [None] * n_pairs
        for i, m in zip(local_ids, local_matches):
            out[i] = np.asarray(m, np.int64).reshape(-1, 2)
        return out
    world, rank = dist.get_world_size(), dist.get_rank()
    dev = device if device is not None else torch.device("cpu")
    k = len(local_ids)
    cnt = torch.tensor([k, max([len(m) for m in local_matches], default=0)], dtype=torch.int64, device=dev)
    cnts = [torch.zeros_like(cnt) for _ in range(world)]
    dist.all_gather(cnts, cnt)
    kmax, smax = int(max(c[0] for c in cnts)), int(max(c[1] for c in cnts))
    buf = torch.full((max(kmax, 1), 2 + 2 * max(smax, 1)), -1, dtype=torch.int64, device=dev)
    for j, (i, m) in enumerate(zip(local_ids, local_matches)):
        m = torch.as_tensor(np.asarray(m, np.int64).reshape(-1, 2), device=dev)
        buf[j, 0], buf[j, 1] = i, m.shape[0]
        if m.shape[0]:
            buf[j, 2:2 + 2 * m.shape[0]] = m.reshape(-1)
    bufs = [torch.zeros_like(buf) for _ in range(world)]
    dist.all_gather(bufs, buf)
    if rank != 0:
        return None
    out = [None] * n_pairs
    for r in range(world):
        b = bufs[r].cpu().numpy()
        for j in range(int(cnts[r][0])):
            i, s = int(b[j, 0]), int(b[j, 1])
            out[i] = b[j, 2:2 + 2 * s].reshape(-1, 2).copy()
    return out


class ImageSetMatcher:
    """Two-phase multi-GPU matching of an image set (module docstring): SuperPoint on this rank's images into the device feature
    store, one all_gather of the float16 feature blocks, LightGlue or SuperGlue on this rank's share of the pair list, gather of the
    match tables.  ``dist`` is ``torch.distributed`` (initialised, nccl) or None for a single process.

    ``matcher="superglue"``: ``lg_weights`` is the SuperGlue state dict and ``lg_conf`` its configuration (``sinkhorn_iterations``,
    ``match_threshold``, ``gnn_layers``), and phase 2 runs the batched device SuperGlue on the store's slots."""

    def __init__(self, ctx, sp_weights: dict, lg_weights: dict, n_images: int, height: int, width: int, sp_conf: dict, lg_conf: dict,
                 batch_images: int = 16, batch_pairs: int = 32, dist=None, matcher: str = "lightglue"):
        import torch

        from . import _native
        self.torch, self.dist, self.ctx = torch, dist, ctx
        self.world = dist.get_world_size() if dist is not None and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world > 1 else 0
        self.n, self.H, self.W = n_images, height, width
        self.cap = int(sp_conf["max_keypoints"])
        self.B, self.P = batch_images, batch_pairs
        self.sp = _native.SuperPointNet(ctx, sp_weights, max_batch=batch_images, max_height=height, max_width=width, **sp_conf)
        if matcher not in ("lightglue", "superglue"):
            raise ValueError(f'matcher must be "lightglue" or "superglue", got {matcher!r}')
        self.matcher = matcher
        if matcher == "superglue":
            self.sg = _native.SuperGlueNet(ctx, lg_weights, max_pairs=batch_pairs, max_kpts=self.cap, **lg_conf)
        else:
            self.lg = _native.LightGlueNet(ctx, lg_weights, max_pairs=batch_pairs, max_kpts=self.cap, **lg_conf)
        self.ipr = images_per_rank(n_images, self.world)
        self.store = _native.FeatureStoreDev(ctx, self.world * self.ipr, self.cap, 256)
        dev = torch.device("cuda", ctx.device)
        # extraction outputs of one batch (float32, library layouts) and match outputs of one pair batch
        self.kp = torch.zeros(batch_images, self.cap, 2, device=dev)
        self.sc = torch.zeros(batch_images, self.cap, device=dev)
        self.de = torch.zeros(batch_images, 256, self.cap, device=dev)
        self.cnt = torch.zeros(batch_images, dtype=torch.int32, device=dev)
        self.m = torch.zeros(batch_pairs, self.cap, 2, dtype=torch.int64, device=dev)
        self.ms = torch.zeros(batch_pairs, self.cap, device=dev)
        self.nm = torch.zeros(batch_pairs, dtype=torch.int32, device=dev)
        self.sl = torch.zeros(batch_pairs, dtype=torch.int32, device=dev)

        class _DevArr:  # zero-copy torch view of the store's device allocation (for the NCCL all_gather)
            def __init__(self, ptr, shape):
                self.__cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": "|u1", "version": 2}

        self.store_t = torch.as_tensor(_DevArr(self.store.base, (self.world * self.ipr, self.store.slot_bytes)), device=dev)
        self.exchanged_bytes = 0

    def extract(self, d_images, image_ids):
        """Phase 1: d_images = float32 CUDA tensor (k, H, W) holding this rank's images `image_ids` (gray 0..255)."""
        st = self.torch.cuda.current_stream().cuda_stream
        for b0 in range(0, len(image_ids), self.B):
            ids = image_ids[b0:b0 + self.B]
            nb = len(ids)
            self.sp.extract_dev(d_images[b0:b0 + nb].data_ptr(), nb, self.H, self.W, self.kp.data_ptr(), self.sc.data_ptr(),
                                self.de.data_ptr(), self.cnt.data_ptr(), self.cap, st)
            for k, i in enumerate(ids):
                self.store.put_dev(store_slot(i, self.n, self.world), self.kp[k].data_ptr(), self.sc[k].data_ptr(), self.de[k].data_ptr(),
                                   self.cap, self.cnt[k:k + 1].data_ptr(), self.H, self.W, None, st)

    def exchange(self):
        """The collective of the path: every rank's float16 feature blocks to every rank (NCCL all_gather over NVLink)."""
        self.exchanged_bytes = all_gather_blocks(self.store_t, self.n, self.dist)

    def match(self, pairs, pair_ids):
        """Phase 2: LightGlue or SuperGlue on `pairs` = [(i, j), ...] (this rank's share); returns {pair id: int64 (S,2)} after ONE
        device->host copy per batch.  Features are read in place from the store (float16, no rounding left to do)."""
        st = self.torch.cuda.current_stream().cuda_stream
        out = {}
        for b0 in range(0, len(pairs), self.P):
            chunk = pairs[b0:b0 + self.P]
            if self.matcher == "superglue":
                f0 = [self.store.sg_feats_dev(store_slot(i, self.n, self.world)) for i, _ in chunk]
                f1 = [self.store.sg_feats_dev(store_slot(j, self.n, self.world)) for _, j in chunk]
                self.sg.match_dev(f0, f1, self.m.data_ptr(), self.ms.data_ptr(), self.nm.data_ptr(), self.cap, st)
            else:
                f0 = [self.store.feats_dev(store_slot(i, self.n, self.world)) for i, _ in chunk]
                f1 = [self.store.feats_dev(store_slot(j, self.n, self.world)) for _, j in chunk]
                self.lg.match_dev(f0, f1, self.m.data_ptr(), self.ms.data_ptr(), self.nm.data_ptr(), self.sl.data_ptr(), self.cap, st)
            nm = self.nm[:len(chunk)].cpu().numpy()
            m = self.m[:len(chunk)].cpu().numpy()
            for k in range(len(chunk)):
                out[pair_ids[b0 + k]] = m[k, :nm[k]].copy()
        return out

    def run(self, d_images, my_image_ids, pairs, costs=None):
        """extract -> exchange -> match my share -> gather to rank 0.  Returns the list of match tables on rank 0 (None elsewhere)."""
        self.extract(d_images, my_image_ids)
        self.exchange()
        mine = shard_pairs(len(pairs), self.world, self.rank, costs)
        res = self.match([pairs[k] for k in mine], mine)
        return gather_match_tables(mine, [res[k] for k in mine], len(pairs), self.dist if self.world > 1 else None,
                                   self.torch.device("cuda", self.ctx.device) if self.world > 1 else None)
