"""One process per GPU: submap-sharded integration and a spatially tiled global map (SURVEY.md section 8e).

* Integration shards by SUBMAP - independent volumes (`ti.root.pointer(ti.i, submap_num)`,
  dense_tsdf.py:116): rank r integrates the frames of the submaps it owns, no data-path collective.
* The GLOBAL map is cut into tiles of whole 16^3 blocks, tile t owned by rank t.  `fuse_submaps_tiled`
  = every rank splats its own submaps, blocks that land in a foreign tile travel to their owner in ONE
  all-to-all (NCCL over NVLink on GPUs) and are reduced there; `exchange_halo` copies the one-block
  boundary layer to the neighbouring tiles as ghost blocks so marching cubes is local; `all_gather_mesh`
  is the final mesh-vertex all-gather.

The collectives are torch.distributed calls on flat tensors, so the bookkeeping below (split sizes, padding,
ownership) is exercised on CPU with the gloo backend (tests/test_distributed_cpu.py) and on GPUs with NCCL
(tests/test_gpu_multi.py, `gpurun --gpus 2`).
"""
import ctypes as C

import numpy as np

from . import _capi as capi


def balanced_tiling(hist, world):
    """Data-driven tiling: `hist` = int[3,1024] marginal histograms of the occupied block coordinates (+512), summed over
    the ranks.  Tries every factorisation tx*ty*tz == world, puts the cuts of each axis at the quantiles of its marginal
    and keeps the factorisation whose heaviest tile (product of the marginal shares) is lightest; ties go to the more
    cubic one.  Returns (tiles, (cuts_x, cuts_y, cuts_z)) with block-coordinate cuts, or (factor_tiles(world), None)
    when nothing is occupied."""
    hist = np.asarray(hist, dtype=np.int64).reshape(3, 1024)
    if hist.sum() == 0:
        return factor_tiles(world), None

    def cuts_for(h, k):
        nz = np.nonzero(h)[0]
        lo, hi = int(nz[0]), int(nz[-1]) + 1
        cs = np.cumsum(h)
        tot = cs[-1]
        cuts = [lo]
        for q in range(1, k):
            c = int(np.searchsorted(cs, tot * q / k, side="left")) + 1  # first coordinate past the q/k quantile
            c = max(c, cuts[-1] + 1)
            cuts.append(c)
        cuts.append(max(hi, cuts[-1] + 1))
        shares = [h[cuts[i]:cuts[i + 1]].sum() / tot for i in range(k)]
        return cuts, max(shares)

    best = None
    for tx in range(1, world + 1):
        if world % tx:
            continue
        for ty in range(1, world // tx + 1):
            if (world // tx) % ty:
                continue
            tz = world // tx // ty
            if max(tx, ty, tz) > 16:
                continue
            cx, sx = cuts_for(hist[0], tx)
            cy, sy = cuts_for(hist[1], ty)
            cz, sz = cuts_for(hist[2], tz)
            score = (round(sx * sy * sz * world, 3), max(tx, ty, tz) - min(tx, ty, tz))
            if best is None or score < best[0]:
                best = (score, (tx, ty, tz), ([c - 512 for c in cx], [c - 512 for c in cy], [c - 512 for c in cz]))
    return best[1], best[2]


def factor_tiles(world):
    """tiles (tx,ty,tz) with tx*ty*tz == world, as cubic as possible, x >= y >= z (8 -> 2x2x2, 4 -> 2x2x1)."""
    best = (world, 1, 1)
    for tx in range(1, world + 1):
        if world % tx:
            continue
        for ty in range(1, world // tx + 1):
            if (world // tx) % ty:
                continue
            tz = world // tx // ty
            cand = tuple(sorted((tx, ty, tz), reverse=True))
            if max(cand) - min(cand) < max(best) - min(best):
                best = cand
    return best


def merge_fuse_plans(rows):
    """Merge of the ranks' plans of a tiled incremental fusion (TiledGlobalMap.update_fused_submaps).  rows: int64
    [world, 3 + 2 S], rank r's row = (full-update reason, cost, cost_full, present[S], include[S]) as
    tslam_tsdf_fuse_update_tiled_plan reports them (present: the rank's collection holds blocks of the submap; include:
    0/1 per submap, all 1 for None).  Returns the reason code every rank splats with: the smallest non-zero reason of
    any rank, else 6 when the summed cost exceeds the summed cost_full (subtracting and re-adding would splat more
    than a rebuild), else 0 (incremental).  Raises ValueError when a submap has blocks on two ranks, or when include
    differs between ranks."""
    rows = np.asarray(rows, dtype=np.int64)
    if rows.ndim != 2 or rows.shape[1] < 3 or (rows.shape[1] - 3) % 2:
        raise ValueError(f"plan rows of shape {rows.shape}: expected [world, 3 + 2 * max_submaps]")
    S = (rows.shape[1] - 3) // 2
    present, include = rows[:, 3:3 + S], rows[:, 3 + S:]
    shared = np.flatnonzero((present != 0).sum(0) > 1)
    if shared.size:
        ranks = [np.flatnonzero(present[:, s]).tolist() for s in shared[:4]]
        raise ValueError(f"tiled fusion: submaps {shared.tolist()} have blocks on several ranks (ranks {ranks}); a submap is "
                         "contributed by one rank")
    if np.any(include != include[:1]):
        raise ValueError("tiled fusion: include differs between ranks (submaps "
                         f"{np.flatnonzero(np.any(include != include[:1], 0)).tolist()}); every rank must pass the same")
    reasons = rows[:, 0]
    if np.any(reasons != 0):
        return int(reasons[reasons != 0].min())
    return 6 if int(rows[:, 1].sum()) > int(rows[:, 2].sum()) else 0


# counters of the tiled incremental fusion, summed over the ranks
_UPDATE_SUMS = ("added", "moved", "removed", "within_tolerance", "voxels_splatted", "voxels_skipped", "blocks_committed",
                "foreign_blocks_sent", "foreign_blocks_received", "bytes_sent")


def _attempt(fn, *args):
    """(0, fn(*args)), or (error code, message) when the library refuses or fails: a phase that fails on one rank must
    still reach the collective where the ranks agree on it."""
    try:
        return 0, fn(*args)
    except capi.TslamError as e:
        return e.code, str(e)


def submap_owner(submap_id, world):
    return int(submap_id) % int(world)


def shard_frames(frame_submaps, rank, world):
    """Indices of the frames whose submap this rank owns."""
    fs = np.asarray(frame_submaps)
    return np.nonzero(fs % world == rank)[0]


def split_offsets(counts):
    counts = np.asarray(counts, dtype=np.int64)
    off = np.zeros(len(counts) + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    return off


def exchange_counts(dist, send_counts, device):
    """all_to_all of one int64 per peer -> how many rows every peer sends to me."""
    import torch
    s = torch.as_tensor(np.asarray(send_counts, dtype=np.int64), device=device)
    r = torch.empty_like(s)
    dist.all_to_all_single(r, s)
    return r.cpu().numpy()


def exchange_rows(dist, tensor, send_counts, recv_counts):
    """all_to_all_single of variable row counts (rows grouped by destination in `tensor`)."""
    import torch
    row = int(np.prod(tensor.shape[1:])) if tensor.dim() > 1 else 1
    flat = tensor.reshape(-1)
    out = torch.empty((int(np.sum(recv_counts)),) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
    dist.all_to_all_single(out.reshape(-1), flat, output_split_sizes=[int(c) * row for c in recv_counts],
                           input_split_sizes=[int(c) * row for c in send_counts])
    return out


def all_gather_ragged(dist, tensor, world):
    """All-gather of per-rank row blocks of different length: counts first, then padded payload (mesh all-gather)."""
    import torch
    n = torch.tensor([tensor.shape[0]], dtype=torch.int64, device=tensor.device)
    counts = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(counts, n)
    counts = [int(c.item()) for c in counts]
    m = max(counts) if counts else 0
    pad = torch.zeros((m,) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
    pad[:tensor.shape[0]] = tensor
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return torch.cat([p[:c] for p, c in zip(parts, counts)], 0), counts


class LocalGroup:
    """Stand-in for torch.distributed inside ONE process: `world` virtual ranks whose TiledGlobalMap objects are driven
    phase by phase (pack on every rank -> route -> unpack on every rank) by run_local_*.  Exercises every pack / unpack
    kernel of csrc/tslam_dist.cu and the whole ownership / split bookkeeping on a single GPU (tests/test_gpu_dist_local.py);
    the NCCL path differs only in who moves the packed rows."""

    def __init__(self, world):
        self.world = int(world)


def _route(send_bufs, send_counts, world):
    """send_bufs[r] = tuple of tensors with rows grouped by destination, send_counts[r][d] rows for d.  Returns per
    destination the tuple of concatenated tensors (source-major, like all_to_all_single) and the receive counts."""
    import torch
    offs = [split_offsets(c) for c in send_counts]
    nbuf = len(send_bufs[0])
    out, rcounts = [], []
    for d in range(world):
        out.append(tuple(torch.cat([send_bufs[r][b][offs[r][d]:offs[r][d + 1]] for r in range(world)], 0) for b in range(nbuf)))
        rcounts.append([int(send_counts[r][d]) for r in range(world)])
    return out, rcounts


class TiledGlobalMap:
    """A DenseTSDF global map whose volume is tiled over the ranks of a torch.distributed group.

    Textured maps (reference: colour is fused with geometry, dense_tsdf.py:276-277) exchange the colour planes too."""

    def __init__(self, global_map, dist, rank, world, tiles=None, balance=True):
        self.m = global_map
        self.dist = dist
        self.rank, self.world = int(rank), int(world)
        self.tiles = tuple(tiles) if tiles is not None else factor_tiles(world)
        self.balance = bool(balance) and tiles is None
        assert self.tiles[0] * self.tiles[1] * self.tiles[2] == self.world
        self._tiles_c = (C.c_int32 * 3)(*self.tiles)
        self.cuts = None
        self.last_exchange = {}
        self._halo_current = False  # ghosts carry the TSDF of the last fusion (exchange_halo ran since)
        self.esdf_submap = 0
        self.last_query = {}  # raycast: dict(rounds, rays_forwarded) of the last batch

    # ---- helpers ----------------------------------------------------------------------------------------
    def _L(self):
        return self.m._h.L

    def _h(self):
        return self.m._h.h

    def owner_of_block(self, bx, by, bz):
        o = C.c_int32(0)
        capi.check(self._L().tslam_tiling_owner(self._h(), self._tiles_c, self.world, int(bx), int(by), int(bz), C.byref(o)))
        return int(o.value)

    def set_tiling(self, tiles, cuts):
        """Install a tiling on this rank (every rank must install the same one)."""
        self.tiles = tuple(int(t) for t in tiles)
        self._tiles_c = (C.c_int32 * 3)(*self.tiles)
        self.cuts = cuts
        if cuts is None:
            capi.check(self._L().tslam_tiling_set_cuts(self._h(), None, None, None, None))
        else:
            arrs = [np.ascontiguousarray(np.asarray(c, dtype=np.int32)) for c in cuts]
            capi.check(self._L().tslam_tiling_set_cuts(self._h(), self._tiles_c, capi.np_ptr(arrs[0]), capi.np_ptr(arrs[1]), capi.np_ptr(arrs[2])))

    # ---- fusion, phase by phase -------------------------------------------------------------------------
    def fusion_splat(self, submaps):
        """Phase 1: splat this rank's submaps (sums pending) and return the marginal histograms of the touched blocks."""
        L, h, st = self._L(), self._h(), capi.stream_ptr()
        submaps._flush()
        capi.check(L.tslam_tsdf_fuse_pending(h, submaps._h.h, st))  # (resets the global map first, dense_tsdf.py:313)
        hist = np.zeros((3, 1024), np.int32)
        capi.check(L.tslam_tsdf_dirty_hist(h, capi.np_ptr(hist), st))
        return hist

    def fusion_pack(self):
        """Phase 2: blocks that fell into a foreign tile -> (send counts, (keys, acc, obs, occ[, col])) grouped by owner."""
        import torch
        L, h, st = self._L(), self._h(), capi.stream_ptr()
        tex = bool(getattr(self.m, "enable_texture", False))
        send, bufs = capi.pack(
            lambda send: L.tslam_tsdf_foreign_count(h, self._tiles_c, self.rank, self.world, send, st),
            lambda send, n, keys, acc, obs, occ, col=None: L.tslam_tsdf_foreign_pack2(h, self._tiles_c, self.rank, self.world, send, n,
                                                                                       keys, acc, obs, occ, col, st),
            self.world, ((), torch.int64), ((4096, 2), torch.float32), ((4096,), torch.uint8), ((4096,), torch.int8),
            *([((4096, 4), torch.float32)] if tex else []))
        n_send = int(send.sum())
        self.last_exchange = {"fusion_blocks_sent": n_send, "fusion_bytes_sent": n_send * (8 + 4096 * (10 + (16 if tex else 0)))}
        return send, bufs

    def fusion_unpack(self, bufs):
        """Phase 3: add the received blocks, commit this rank's tile."""
        import torch
        L, h, st = self._L(), self._h(), capi.stream_ptr()
        n_recv = int(bufs[0].shape[0])
        col = bufs[4] if len(bufs) > 4 else None
        capi.check(L.tslam_tsdf_unpack_add2(h, n_recv, capi.tptr(bufs[0]), capi.tptr(bufs[1]), capi.tptr(bufs[2]), capi.tptr(bufs[3]),
                                            capi.tptr(col), st))
        capi.check(L.tslam_tsdf_commit_fused(h, st))
        torch.cuda.current_stream().synchronize()  # received buffers must outlive the kernels
        self.last_exchange["fusion_blocks_received"] = n_recv
        self._halo_current = False

    def fuse_submaps_tiled(self, submaps):
        """fuse_submaps (dense_tsdf.py:312-318) with the result tiled over the ranks.  `submaps` = this rank's
        submap collection; the pose table of the global map must hold the poses of the submaps it contains."""
        import torch
        dev = capi.device()
        hist = self.fusion_splat(submaps)
        if self.balance:
            ht = torch.as_tensor(hist.astype(np.int64), device=dev)
            self.dist.all_reduce(ht)
            tiles, cuts = balanced_tiling(ht.cpu().numpy(), self.world)
            self.set_tiling(tiles, cuts)
        send, bufs = self.fusion_pack()
        recv = exchange_counts(self.dist, send, dev)
        rbufs = tuple(exchange_rows(self.dist, b, send, recv) for b in bufs)
        self.fusion_unpack(rbufs)

    # ---- incremental fusion with exact integer sums, phase by phase (csrc/tslam_fuse.cu) -------------------------
    # The contract is tslam_tsdf_fuse_update_tiled_plan's (include/tslam.h, DESIGN.md section 6): the sums of a block live
    # on its owner, the other ranks send integer deltas, so the union of the tiles is bit for bit the single-map
    # tslam_tsdf_fuse_update of every rank's submaps.  update_fused_submaps (NCCL / gloo) and
    # run_local_update_fused_submaps (LocalGroup) run the same phases.
    def update_plan(self, submaps, include=None, tolerance=0.0, full=False):
        """Phase 1: this rank's plan row (merge_fuse_plans) for its submap collection `submaps`."""
        submaps._flush()
        h = self.m._h
        plan, present = h.fuse_update_tiled_plan(submaps._h, self.tiles, self.rank, self.world, include, tolerance, full)
        inc = h.include_u8(include)
        inc = np.ones(present.shape[0], np.int64) if inc is None else inc.astype(np.int64)
        return np.concatenate([plan, present.astype(np.int64), inc])

    def update_splat(self, submaps, reason):
        """Phase 2: splat with the merged reason.  A full update with balanced cuts returns the marginal histograms of
        the blocks its additions activated (to be summed over the ranks for balanced_tiling), else None."""
        self.m._h.fuse_update_tiled_splat(submaps._h, reason)
        if not (reason and self.balance):
            return None
        hist = np.zeros((3, 1024), np.int32)
        capi.check(self._L().tslam_tsdf_dirty_hist(self._h(), capi.np_ptr(hist), capi.stream_ptr()))
        return hist

    def update_pack(self):
        """Phase 3: the sum rows of the foreign blocks -> (send counts, (rows,)) grouped by owner."""
        send, rows = self.m._h.fuse_update_tiled_pack(self.tiles, self.rank, self.world)
        self.last_exchange = {"foreign_blocks_sent": int(send.sum()), "bytes_sent": int(rows.numel()) * 8}
        return send, (rows,)

    def update_unpack(self, bufs):
        """Phase 4: add the received rows into the owned sums and commit the touched blocks."""
        self.m._h.fuse_update_tiled_unpack(bufs[0])
        self.last_exchange["foreign_blocks_received"] = int(bufs[0].shape[0])

    def update_finish(self, submaps, ok):
        """Phase 5: record the update (ok: every rank's phases succeeded) -> this rank's statistics, or None."""
        self._halo_current = False
        st = self.m._h.fuse_update_tiled_finish(submaps._h, ok)
        if st is not None:
            for k in ("foreign_blocks_sent", "foreign_blocks_received", "bytes_sent"):
                st[k] = int(self.last_exchange.get(k, 0))
        return st

    def _agree(self, submaps, rc, msg, dev):
        """Every rank learns whether a phase failed anywhere; if so every rank abandons the update and raises."""
        import torch
        t = torch.tensor([int(rc)], dtype=torch.int64, device=dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MIN)
        worst = int(t.item())
        if worst:
            self.update_finish(submaps, False)
            raise capi.TslamError(worst, msg if rc else "tiled fusion update failed on another rank")

    def update_fused_submaps(self, submaps, include=None, tolerance=0.0, full=False):
        """Incremental fusion of every rank's submaps into the tiled global map (collective; the tiled counterpart of
        TsdfHandle.fuse_update).  `submaps` = this rank's submap collection, include / tolerance / full as fuse_update's
        (include must be the same on every rank); the pose table of every rank's global map holds the poses of all
        submaps.  Afterwards the union of the ranks' tiles is bit for bit the single-map fuse_update of all submaps.
        Only a full update with balanced cuts moves the cuts.  Returns fuse_update's statistics summed over the ranks
        (reason: the same on every rank) plus foreign_blocks_sent / _received and bytes_sent."""
        import torch
        dev = capi.device()
        self.last_exchange = {}
        width = 3 + 2 * capi.submap_table(self.m._h.cfg.max_submaps)
        rc, row = _attempt(self.update_plan, submaps, include, tolerance, full)
        mine = torch.as_tensor(np.concatenate([[rc], row if rc == 0 else np.zeros(width, np.int64)]), dtype=torch.int64, device=dev)
        parts = [torch.empty_like(mine) for _ in range(self.world)]
        self.dist.all_gather(parts, mine)
        rows = torch.stack(parts).cpu().numpy()
        if np.any(rows[:, 0] != 0):
            self.update_finish(submaps, False)
            raise capi.TslamError(int(rows[:, 0].min()), row if rc else "tiled fusion plan failed on another rank")
        try:
            reason = merge_fuse_plans(rows[:, 1:])
        except ValueError:
            self.update_finish(submaps, False)
            raise
        rc, hist = _attempt(self.update_splat, submaps, reason)
        self._agree(submaps, rc, hist, dev)
        if hist is not None:
            ht = torch.as_tensor(hist.astype(np.int64), device=dev)
            self.dist.all_reduce(ht)
            self.set_tiling(*balanced_tiling(ht.cpu().numpy(), self.world))
        rc, packed = _attempt(self.update_pack)
        self._agree(submaps, rc, packed, dev)
        send, bufs = packed
        recv = exchange_counts(self.dist, send, dev)
        rc, msg = _attempt(self.update_unpack, tuple(exchange_rows(self.dist, b, send, recv) for b in bufs))
        self._agree(submaps, rc, msg, dev)
        st = self.update_finish(submaps, True)
        tot = torch.tensor([st[k] for k in _UPDATE_SUMS], dtype=torch.int64, device=dev)
        self.dist.all_reduce(tot)
        st.update(zip(_UPDATE_SUMS, (int(x) for x in tot.cpu().numpy())))
        return st

    # ---- halo + mesh --------------------------------------------------------------------------------------
    def halo_pack(self):
        import torch
        L, h, st = self._L(), self._h(), capi.stream_ptr()
        tex = bool(getattr(self.m, "enable_texture", False))
        send, bufs = capi.pack(
            lambda send: L.tslam_tsdf_halo_count(h, self._tiles_c, self.rank, self.world, send, st),
            lambda send, n, keys, tw, obs, col=None: L.tslam_tsdf_halo_pack2(h, self._tiles_c, self.rank, self.world, send, n, keys, tw,
                                                                              obs, col, st),
            self.world, ((), torch.int64), ((4096, 2), torch.float32), ((4096,), torch.uint8), *([((4096, 4), torch.float32)] if tex else []))
        self.last_exchange["halo_blocks_sent"] = int(send.sum())
        return send, bufs

    def halo_unpack(self, bufs):
        import torch
        L, h, st = self._L(), self._h(), capi.stream_ptr()
        n_recv = int(bufs[0].shape[0])
        col = bufs[3] if len(bufs) > 3 else None
        capi.check(L.tslam_tsdf_ghost_unpack2(h, n_recv, capi.tptr(bufs[0]), capi.tptr(bufs[1]), capi.tptr(bufs[2]), capi.tptr(col), st))
        torch.cuda.current_stream().synchronize()
        self.last_exchange["halo_blocks_received"] = n_recv
        self._halo_current = True

    def exchange_halo(self):
        dev = capi.device()
        send, bufs = self.halo_pack()
        recv = exchange_counts(self.dist, send, dev)
        self.halo_unpack(tuple(exchange_rows(self.dist, b, send, recv) for b in bufs))

    def local_mesh(self, mesher, step=1):
        """Two-pass marching cubes on this rank's tile (+ghosts): triangles of OWNED blocks only."""
        mesher.generate_mesh(step)
        n = min(int(mesher.num_facelets[None]), mesher.max_triangles)
        return mesher.mesh_vertices.t[:3 * n], mesher.mesh_normals.t[:3 * n]

    def generate_mesh_all_gather(self, mesher, step=1):
        """Local two-pass marching cubes on this rank's tile (+ghosts), then the mesh-vertex all-gather."""
        self.exchange_halo()
        v, nrm = self.local_mesh(mesher, step)
        allv, counts = all_gather_ragged(self.dist, v, self.world)
        alln, _ = all_gather_ragged(self.dist, nrm, self.world)
        return allv, alln, [c // 3 for c in counts]


    # ---- ESDF, phase by phase (csrc/tslam_esdf.cu: tslam_esdf_tiled_*) -------------------------------------------
    # The tiled ESDF is a full recompute: begin seeds owned and ghost blocks and runs the local wave with the ghosts as
    # read-only sources; then rounds of (pack the boundary blocks that changed -> all-to-all -> unpack into the
    # neighbours' ghosts -> relax from them) until no rank packs anything.  The result is bit-identical to one map
    # holding every tile (DESIGN.md section 6).
    def esdf_begin(self, submap=0):
        self.esdf_submap = int(submap)
        return self.m._h.esdf_tiled_begin(submap)

    def esdf_halo_pack(self):
        """Owned boundary blocks whose ESDF changed since they were last packed -> (send counts, (keys, esdf))."""
        import torch
        L, h, st = self._L(), self._h(), capi.stream_ptr()
        send, bufs = capi.pack(
            lambda send: L.tslam_esdf_halo_count(h, self._tiles_c, self.rank, self.world, send, st),
            lambda send, n, keys, esdf: L.tslam_esdf_halo_pack(h, self._tiles_c, self.rank, self.world, send, n, keys, esdf, st),
            self.world, ((), torch.int64), ((4096,), torch.float32))
        self.last_exchange["esdf_blocks_sent"] = self.last_exchange.get("esdf_blocks_sent", 0) + int(send.sum())
        return send, bufs

    def esdf_halo_unpack(self, bufs):
        import torch
        self.m._h.esdf_ghost_unpack(bufs[0], bufs[1])
        torch.cuda.current_stream().synchronize()

    def esdf_relax(self):
        return self.m._h.esdf_tiled_relax()

    def esdf_end(self):
        self.m._h.esdf_tiled_end()

    def esdf_update(self, submap=0, max_rounds=1024):
        """Tiled ESDF of `submap` on every rank (collective) -> dict(rounds, sweeps, blocks_sent, bytes_sent) of this
        rank; rounds = exchange rounds in which some rank sent a block.  Runs a TSDF halo exchange first unless one
        has run since the last fusion.  Raises after `max_rounds` rounds."""
        import torch
        dev = capi.device()
        if not self._halo_current:
            self.exchange_halo()
        self.last_exchange["esdf_blocks_sent"] = 0
        sweeps = self.esdf_begin(submap)
        rounds = 0
        while True:
            send, bufs = self.esdf_halo_pack()
            tot = torch.tensor([int(send.sum())], dtype=torch.int64, device=dev)
            self.dist.all_reduce(tot)
            if int(tot.item()) == 0:
                break
            rounds += 1
            if rounds > max_rounds:
                raise RuntimeError(f"tiled ESDF: still exchanging after {max_rounds} rounds")
            recv = exchange_counts(self.dist, send, dev)
            self.esdf_halo_unpack(tuple(exchange_rows(self.dist, b, send, recv) for b in bufs))
            sweeps += self.esdf_relax()
        self.esdf_end()
        return _esdf_stats(rounds, sweeps, self.last_exchange["esdf_blocks_sent"])

    def _query_dest(self, xyz):
        """Points f32[n,3] on the device and the rank that answers each: the owner of the block holding its low
        interpolation corner; this rank for points no tile holds (they come out invalid anywhere)."""
        return capi.owner_ranks(self._L().tslam_tiling_owner_points, self._h(), self._tiles_c, self.world, self.rank, xyz)

    def _esdf_answer(self, pts):
        """tslam_esdf_query on points routed here -> (dist|grad f32[n,4], valid u8[n])."""
        import torch
        n = pts.shape[0]
        dg = torch.empty((n, 4), dtype=torch.float32, device=pts.device)
        dist = torch.empty(n, dtype=torch.float32, device=pts.device)
        grad = torch.empty((n, 3), dtype=torch.float32, device=pts.device)
        valid = torch.empty(n, dtype=torch.uint8, device=pts.device)
        capi.check(self._L().tslam_esdf_query(self._h(), self.esdf_submap, n, capi.tptr(pts), capi.tptr(dist), capi.tptr(grad),
                                              capi.tptr(valid), capi.stream_ptr()))
        dg[:, 0] = dist
        dg[:, 1:] = grad
        return dg, valid

    def esdf_query(self, xyz):
        """Trilinear ESDF and gradient (TsdfHandle.esdf_query) at this rank's points, answered by the ranks that own
        them (collective: every rank calls it, with any points).  Returns (dist, grad, valid) in the caller's order:
        torch CUDA tensors for a torch tensor, numpy arrays for numpy."""
        import torch
        as_torch = isinstance(xyz, torch.Tensor)
        x, dest = self._query_dest(xyz)
        dg, valid = routed_answers(self.dist, x, dest, self.world, self._esdf_answer)
        return _query_result(dg, valid, as_torch)

    def esdf_slice_local(self, z):
        """This rank's part of the ESDF slice at height z: (xyz f32[n,3], ESDF f32[n]) torch CUDA tensors."""
        import torch
        dev = capi.device()
        _, xyz, val = self.m._h.esdf_slice(z, submap=self.esdf_submap)
        return torch.from_numpy(xyz).to(dev), torch.from_numpy(val).to(dev)

    def esdf_slice_all_gather(self, z):
        """cvt_ESDF_to_voxels_slice of the whole tiled map on every rank: (xyz, ESDF) torch CUDA tensors."""
        xyz, val = self.esdf_slice_local(z)
        allx, _ = all_gather_ragged(self.dist, xyz, self.world)
        allv, _ = all_gather_ragged(self.dist, val, self.world)
        return allx, allv

    # ---- planner queries: BaseMap's surface (mapping_common.py:165-204) on the tiled map ---------------------------
    # Collectives: every rank calls them, with any points (an empty batch included); the answers come back in the
    # caller's order and are bit-identical to the same call on one DenseTSDF holding every tile (DESIGN.md section 6).
    # TopoGraphGen(tiled) therefore works unchanged when every rank runs the same TopoGraphGen in lockstep: its host
    # code is deterministic numpy, so the ranks issue identical calls.
    @property
    def voxel_scale(self):
        return self.m.voxel_scale

    def ray_round_bound(self):
        """Hand-over rounds a raycast batch can need: one into the tile of the first sample, then one per tile change,
        at most tiles - 1 per axis because the tile of a ray's samples is monotone on each axis."""
        return sum(self.tiles) - 2

    def _ray_rows(self, pos, dir, max_dist):
        """Rays f32[n,8] (pos, dir, max_dist, next sample 0) and their tags row * world + rank (int64[n])."""
        import torch
        p, d = capi.to_device(pos, (-1, 3)), capi.to_device(dir, (-1, 3))
        rays = torch.zeros((p.shape[0], 8), dtype=torch.float32, device=p.device)  # (j = 0: int32 0 has the bits of 0.0f)
        rays[:, :3] = p
        rays[:, 3:6] = d
        rays[:, 6] = float(max_dist)
        return rays, torch.arange(p.shape[0], dtype=torch.int64, device=p.device) * self.world + self.rank

    def _march(self, rays):
        """One round of tslam_tsdf_raycast_tiled on the rays held here -> (dest int64[n], answer f32[n,5] = hit,
        xyz, len; meaningful where dest < 0)."""
        import torch
        n, dev = rays.shape[0], rays.device
        dest = torch.empty(n, dtype=torch.int32, device=dev)
        hit = torch.empty(n, dtype=torch.uint8, device=dev)
        xyz = torch.empty((n, 3), dtype=torch.float32, device=dev)
        ln = torch.empty(n, dtype=torch.float32, device=dev)
        capi.check(self._L().tslam_tsdf_raycast_tiled(self._h(), self._tiles_c, self.rank, self.world, self.m._active(), n, capi.tptr(rays),
                                                      capi.tptr(dest), capi.tptr(hit), capi.tptr(xyz), capi.tptr(ln), capi.stream_ptr()))
        return dest.long(), torch.cat([hit.float()[:, None], xyz, ln[:, None]], 1)

    def _cell_dest(self, xyz):
        """Points f32[n,3] on the device and the rank that answers each: the owner of the block holding its cell; this
        rank for cells outside the volume (occupied and unobserved anywhere)."""
        return capi.owner_ranks(self._L().tslam_tiling_owner_cells, self._h(), self._tiles_c, self.world, self.rank, xyz)

    def _points_answer(self, pts):
        """tslam_tsdf_query_points on points routed here -> (flags u8[n],)."""
        import torch
        f = torch.empty(pts.shape[0], dtype=torch.uint8, device=pts.device)
        capi.check(self._L().tslam_tsdf_query_points(self._h(), self.m._active(), pts.shape[0], capi.tptr(pts), capi.tptr(f), capi.stream_ptr()))
        return (f,)

    def _near_answer(self, pts, voxel):
        """tslam_tsdf_query_near_occupy_tiled (reads ghosts) on points routed here -> (u8[n],)."""
        import torch
        f = torch.empty(pts.shape[0], dtype=torch.uint8, device=pts.device)
        capi.check(self._L().tslam_tsdf_query_near_occupy_tiled(self._h(), self.m._active(), pts.shape[0], capi.tptr(pts), int(voxel), capi.tptr(f),
                                                                capi.stream_ptr()))
        return (f,)

    def raycast(self, pos, dir, max_dist):
        """BaseMap.raycast: (succ, last position, length) per ray, each ray marched by the ranks whose tiles it crosses.
        self.last_query = dict(rounds, rays_forwarded) (summed over the ranks)."""
        from .mapping.mapping_common import BaseMap
        p, single = BaseMap._as_batch(pos)
        d, _ = BaseMap._as_batch(dir)
        rays, tags = self._ray_rows(p, d, max_dist)
        (ans,), self.last_query = raycast_rounds(_DistRouter(self.dist, self.world, rays.device), [self._march], [rays], [tags], self.world,
                                                 self.ray_round_bound())
        return _ray_result(ans, single)

    def _query_points(self, xyz):
        x, dest = self._cell_dest(xyz)
        (f,) = routed_answers(self.dist, x, dest, self.world, self._points_answer)
        f = f.cpu().numpy()
        return (f & 1).astype(bool), (f & 2).astype(bool)

    def is_pos_occupy(self, xyz):
        from .mapping.mapping_common import BaseMap
        p, single = BaseMap._as_batch(xyz)
        r = self._query_points(p)[0]
        return bool(r[0]) if single else r

    def is_pos_unobserved(self, xyz):
        from .mapping.mapping_common import BaseMap
        p, single = BaseMap._as_batch(xyz)
        r = self._query_points(p)[1]
        return bool(r[0]) if single else r

    def is_near_pos_occupy(self, xyz, voxel):
        """Answered by the owner of the centre cell, reading its ghosts: runs a TSDF halo exchange first unless one
        has run since the last fusion.  voxel must lie in [0, 16] (the halo is one block deep)."""
        from .mapping.mapping_common import BaseMap
        voxel = _near_voxel(voxel)
        p, single = BaseMap._as_batch(xyz)
        if not self._halo_current:
            self.exchange_halo()
        x, dest = self._cell_dest(p)
        (f,) = routed_answers(self.dist, x, dest, self.world, lambda pts: self._near_answer(pts, voxel))
        r = f.cpu().numpy().astype(bool)
        return bool(r[0]) if single else r


def _esdf_stats(rounds, sweeps, blocks):
    return dict(rounds=int(rounds), sweeps=int(sweeps), blocks_sent=int(blocks), bytes_sent=int(blocks) * (8 + 4096 * 4))


def _query_result(dg, valid, as_torch):
    import torch
    dist, grad, valid = dg[:, 0].contiguous(), dg[:, 1:].contiguous(), valid.view(torch.bool)
    if as_torch:
        return dist, grad, valid
    return dist.cpu().numpy(), grad.cpu().numpy(), valid.cpu().numpy()


def route_order(dest, world):
    """Rows addressed to ranks dest (int64 tensor [n]): the stable order that groups them by destination, and the
    rows per destination."""
    import torch
    order = torch.argsort(dest, stable=True)
    counts = torch.bincount(dest, minlength=world).cpu().numpy().astype(np.int64)
    return order, counts


def route_restore(order, rows):
    """Undo route_order: rows[i] belongs to caller row order[i]."""
    import torch
    out = torch.empty_like(rows)
    out[order] = rows
    return out


def routed_answers(dist, rows, dest, world, answer):
    """Send row i to rank dest[i] (all-to-all), answer there with answer(rows) -> tuple of tensors with one row per
    row, send the answers back: the answers in the caller's row order."""
    order, send = route_order(dest, world)
    recv = exchange_counts(dist, send, rows.device)
    got = exchange_rows(dist, rows[order], send, recv)
    return tuple(route_restore(order, exchange_rows(dist, a, recv, send)) for a in answer(got))


class _DistRouter:
    """The ranks of a torch.distributed group, one per process: raycast_rounds sees a list of one local rank."""

    def __init__(self, dist, world, device):
        self.dist, self.world, self.device = dist, int(world), device

    def total(self, counts):
        import torch
        t = torch.tensor([int(sum(counts))], dtype=torch.int64, device=self.device)
        self.dist.all_reduce(t)
        return int(t.item())

    def route(self, bufs, dests):
        """bufs[0] = tuple of tensors, row i addressed to rank dests[0][i] -> [tuple of the rows received]."""
        order, send = route_order(dests[0], self.world)
        recv = exchange_counts(self.dist, send, self.device)
        return [tuple(exchange_rows(self.dist, b[order], send, recv) for b in bufs[0])]


class _LocalRouter:
    """`world` virtual ranks in one process (LocalGroup): the all-to-all is _route's slicing."""

    def __init__(self, world):
        self.world = int(world)

    def total(self, counts):
        return int(sum(counts))

    def route(self, bufs, dests):
        orders, sends = zip(*[route_order(d, self.world) for d in dests])
        routed, _ = _route([tuple(b[o] for b in bb) for bb, o in zip(bufs, orders)], sends, self.world)
        return routed


def raycast_rounds(router, marches, rays, tags, world, bound):
    """The hand-over loop of a routed raycast over the local ranks k of `router` (one per process with NCCL / gloo,
    all of them for LocalGroup).  rays[k] f32[n,8] and tags[k] int64[n] (row * world + origin rank) are rank k's
    rays; marches[k](rays) -> (dest int64[n], answer f32[n,5]) marches them as far as rank k's tile goes (dest -1:
    finished, with its answer).  Rounds: march, count the handed-over rays over all ranks, stop at 0, route them to
    their dest.  Raises past `bound` rounds, which the tile monotonicity of a ray rules out (DESIGN.md section 6).
    Finally every answer goes home in one exchange.  Returns ([answer f32[n_k,5] in rank k's row order], dict(rounds,
    rays_forwarded) summed over the ranks)."""
    import torch
    n0 = [int(r.shape[0]) for r in rays]
    rays, tags = list(rays), list(tags)
    fin_tags, fin_ans = [[] for _ in rays], [[] for _ in rays]
    rounds = forwarded = 0
    while True:
        dests = []
        for k, march in enumerate(marches):
            dest, ans = march(rays[k])
            done = dest < 0
            fin_tags[k].append(tags[k][done])
            fin_ans[k].append(ans[done])
            rays[k], tags[k] = rays[k][~done], tags[k][~done]
            dests.append(dest[~done])
        n = router.total([int(d.shape[0]) for d in dests])
        if n == 0:
            break
        rounds += 1
        if rounds > bound:
            raise RuntimeError(f"tiled raycast: rays still handed over after {bound} rounds (the bound of a tiling {world} wide)")
        forwarded += n
        got = router.route([(r, t) for r, t in zip(rays, tags)], dests)
        rays, tags = [g[0] for g in got], [g[1] for g in got]
    tags = [torch.cat(t) for t in fin_tags]
    home = router.route([(torch.cat(a), t) for a, t in zip(fin_ans, tags)], [t % world for t in tags])
    out = []
    for n, (ans, tag) in zip(n0, home):
        o = torch.empty((n, 5), dtype=ans.dtype, device=ans.device)
        o[tag // world] = ans
        out.append(o)
    return out, dict(rounds=rounds, rays_forwarded=forwarded)


def _ray_result(ans, single):
    """answer f32[n,5] of raycast_rounds -> BaseMap.raycast's (succ, xyz, len)."""
    a = ans.cpu().numpy()
    succ, xyz, ln = a[:, 0] > 0, np.ascontiguousarray(a[:, 1:4]), np.ascontiguousarray(a[:, 4])
    return (bool(succ[0]), xyz[0], float(ln[0])) if single else (succ, xyz, ln)


def _near_voxel(voxel):
    voxel = int(voxel)
    if not 0 <= voxel <= 16:
        raise ValueError(f"is_near_pos_occupy on a tiled map: voxel {voxel} outside [0, 16] (the halo is one 16^3 block deep)")
    return voxel


def run_local_fusion(tiled, submaps):
    """Tiled fusion of `world` virtual ranks living in ONE process: tiled[r] / submaps[r] = rank r's global map wrapper
    and submap collection.  Same phases as TiledGlobalMap.fuse_submaps_tiled, the all-to-all replaced by slicing."""
    world = len(tiled)
    hists = [t.fusion_splat(s) for t, s in zip(tiled, submaps)]
    if tiled[0].balance:
        tiles, cuts = balanced_tiling(np.sum([h.astype(np.int64) for h in hists], axis=0), world)
        for t in tiled:
            t.set_tiling(tiles, cuts)
    packed = [t.fusion_pack() for t in tiled]
    routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], world)
    for t, bufs in zip(tiled, routed):
        t.fusion_unpack(bufs)


def run_local_update_fused_submaps(tiled, submaps, include=None, tolerance=0.0, full=False):
    """TiledGlobalMap.update_fused_submaps on `world` virtual ranks in one process: tiled[r] / submaps[r] = rank r's
    global map wrapper and submap collection, the all-to-all replaced by slicing.  Returns the statistics summed over
    the ranks."""
    world = len(tiled)
    for t in tiled:
        t.last_exchange = {}

    def agree(res):
        bad = [(rc, msg) for rc, msg in res if rc]
        if bad:
            for t, s in zip(tiled, submaps):
                t.update_finish(s, False)
            raise capi.TslamError(min(rc for rc, _ in bad), bad[0][1])
        return [r for _, r in res]

    rows = agree([_attempt(t.update_plan, s, include, tolerance, full) for t, s in zip(tiled, submaps)])
    try:
        reason = merge_fuse_plans(np.stack(rows))
    except ValueError:
        for t, s in zip(tiled, submaps):
            t.update_finish(s, False)
        raise
    hists = agree([_attempt(t.update_splat, s, reason) for t, s in zip(tiled, submaps)])
    if hists[0] is not None:
        tiles, cuts = balanced_tiling(np.sum([h.astype(np.int64) for h in hists], axis=0), world)
        for t in tiled:
            t.set_tiling(tiles, cuts)
    packed = agree([_attempt(t.update_pack) for t in tiled])
    routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], world)
    agree([_attempt(t.update_unpack, b) for t, b in zip(tiled, routed)])
    stats = [t.update_finish(s, True) for t, s in zip(tiled, submaps)]
    out = dict(stats[0])
    for k in _UPDATE_SUMS:
        out[k] = sum(st[k] for st in stats)
    return out


def run_local_mesh(tiled, meshers, step=1):
    world = len(tiled)
    packed = [t.halo_pack() for t in tiled]
    routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], world)
    for t, bufs in zip(tiled, routed):
        t.halo_unpack(bufs)
    import torch
    vs, ns = zip(*[t.local_mesh(m, step) for t, m in zip(tiled, meshers)])
    return torch.cat(vs, 0), torch.cat(ns, 0), [int(v.shape[0]) // 3 for v in vs]


def run_local_esdf(tiled, submap=0, max_rounds=1024):
    """TiledGlobalMap.esdf_update on `world` virtual ranks in one process; the statistics are summed over the ranks."""
    world = len(tiled)
    if not all(t._halo_current for t in tiled):
        packed = [t.halo_pack() for t in tiled]
        routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], world)
        for t, bufs in zip(tiled, routed):
            t.halo_unpack(bufs)
    sweeps = sum(t.esdf_begin(submap) for t in tiled)
    rounds = blocks = 0
    while True:
        packed = [t.esdf_halo_pack() for t in tiled]
        n = sum(int(p[0].sum()) for p in packed)
        if n == 0:
            break
        rounds += 1
        blocks += n
        if rounds > max_rounds:
            raise RuntimeError(f"tiled ESDF: still exchanging after {max_rounds} rounds")
        routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], world)
        for t, bufs in zip(tiled, routed):
            t.esdf_halo_unpack(bufs)
        sweeps += sum(t.esdf_relax() for t in tiled)
    for t in tiled:
        t.esdf_end()
    return _esdf_stats(rounds, sweeps, blocks)


def run_local_esdf_query(tiled, xyz_per_rank):
    """TiledGlobalMap.esdf_query on `world` virtual ranks: [(dist, grad, valid)] per rank, in each caller's order."""
    import torch
    world = len(tiled)
    plans = [t._query_dest(x) for t, x in zip(tiled, xyz_per_rank)]
    orders, sends = zip(*[route_order(dest, world) for _, dest in plans])
    routed, rcounts = _route([(x[o],) for (x, _), o in zip(plans, orders)], sends, world)
    answers = [t._esdf_answer(pts[0]) for t, pts in zip(tiled, routed)]
    back, _ = _route(answers, rcounts, world)
    return [_query_result(route_restore(o, b[0]), route_restore(o, b[1]), isinstance(x, torch.Tensor))
            for o, b, x in zip(orders, back, xyz_per_rank)]


def run_local_raycast(tiled, rays_per_rank):
    """TiledGlobalMap.raycast on `world` virtual ranks: rays_per_rank[r] = (pos, dir, max_dist) of rank r ->
    [(succ, xyz, len)] per rank in each caller's order; every tiled[r].last_query = dict(rounds, rays_forwarded)."""
    from .mapping.mapping_common import BaseMap
    world = len(tiled)
    rows = [t._ray_rows(BaseMap._as_batch(p)[0], BaseMap._as_batch(d)[0], m) for t, (p, d, m) in zip(tiled, rays_per_rank)]
    ans, st = raycast_rounds(_LocalRouter(world), [t._march for t in tiled], [r[0] for r in rows], [r[1] for r in rows], world,
                             tiled[0].ray_round_bound())
    for t in tiled:
        t.last_query = dict(st)
    return [_ray_result(a, False) for a in ans]


def _run_local_routed(tiled, xyz_per_rank, answer):
    """Points of every virtual rank routed to the owners of their cells, answered there by answer(t, pts) -> (u8[n],),
    and sent back: [u8 numpy array] per rank in each caller's order."""
    world = len(tiled)
    plans = [t._cell_dest(x) for t, x in zip(tiled, xyz_per_rank)]
    orders, sends = zip(*[route_order(dest, world) for _, dest in plans])
    routed, rcounts = _route([(x[o],) for (x, _), o in zip(plans, orders)], sends, world)
    back, _ = _route([answer(t, pts[0]) for t, pts in zip(tiled, routed)], rcounts, world)
    return [route_restore(o, b[0]).cpu().numpy() for o, b in zip(orders, back)]


def run_local_query_points(tiled, xyz_per_rank):
    """is_pos_occupy / is_pos_unobserved on `world` virtual ranks -> [(occupied, unobserved)] per rank."""
    f = _run_local_routed(tiled, xyz_per_rank, lambda t, pts: t._points_answer(pts))
    return [((a & 1).astype(bool), (a & 2).astype(bool)) for a in f]


def run_local_near_occupy(tiled, xyz_per_rank, voxel):
    """is_near_pos_occupy on `world` virtual ranks (halo exchange first unless current) -> [bool array] per rank."""
    voxel = _near_voxel(voxel)
    world = len(tiled)
    if not all(t._halo_current for t in tiled):
        packed = [t.halo_pack() for t in tiled]
        routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], world)
        for t, bufs in zip(tiled, routed):
            t.halo_unpack(bufs)
    return [a.astype(bool) for a in _run_local_routed(tiled, xyz_per_rank, lambda t, pts: t._near_answer(pts, voxel))]


class LocalGroupMap:
    """BaseMap's planner-query surface over the `world` virtual ranks of a LocalGroup (tiled[r] = rank r's
    TiledGlobalMap), so that TopoGraphGen runs on a tiled map on one GPU.  Every query is asked by virtual rank
    `asker`; the other ranks take part with empty batches, as ranks with nothing to ask do under NCCL."""

    def __init__(self, tiled, asker=0):
        self.tiled, self.asker = list(tiled), int(asker)
        self.voxel_scale = self.tiled[0].voxel_scale
        self.last_query = {}

    def _per_rank(self, a):
        empty = np.zeros((0, 3), np.float32)
        return [a if r == self.asker else empty for r in range(len(self.tiled))]

    def raycast(self, pos, dir, max_dist):
        from .mapping.mapping_common import BaseMap
        p, single = BaseMap._as_batch(pos)
        d, _ = BaseMap._as_batch(dir)
        out = run_local_raycast(self.tiled, [(a, b, max_dist) for a, b in zip(self._per_rank(p), self._per_rank(d))])[self.asker]
        self.last_query = dict(self.tiled[0].last_query)
        succ, xyz, ln = out
        return (bool(succ[0]), xyz[0], float(ln[0])) if single else out

    def _points(self, xyz, bit):
        from .mapping.mapping_common import BaseMap
        p, single = BaseMap._as_batch(xyz)
        r = run_local_query_points(self.tiled, self._per_rank(p))[self.asker][bit]
        return bool(r[0]) if single else r

    def is_pos_occupy(self, xyz):
        return self._points(xyz, 0)

    def is_pos_unobserved(self, xyz):
        return self._points(xyz, 1)

    def is_near_pos_occupy(self, xyz, voxel):
        from .mapping.mapping_common import BaseMap
        p, single = BaseMap._as_batch(xyz)
        r = run_local_near_occupy(self.tiled, self._per_rank(p), voxel)[self.asker]
        return bool(r[0]) if single else r
