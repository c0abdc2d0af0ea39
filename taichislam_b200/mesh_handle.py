"""MeshCache - the incremental marching-cubes mesh of one map (tslam_mesh_*, include/tslam.h).

update() gives what tslam_mc_generate2(step=1) gives, bit for bit, while remeshing only the blocks a commit since the
previous update could have changed.  Outputs are torch CUDA tensors written on the current stream.
"""
import ctypes as C

from . import _capi as capi


class MeshCache:
    def __init__(self, handle):
        """handle: the TsdfHandle of the map.  The cache keeps it alive: a cache must go before its map."""
        self.map = handle
        self.L = handle.L
        h = C.c_void_p()
        capi.check(self.L.tslam_mesh_create(handle.h, C.byref(h)))
        self.h = h
        self.stats = (0, 0, 0, 0)

    def close(self):
        if getattr(self, "h", None):
            self.L.tslam_mesh_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def update_into(self, thres, cap_tri, verts, normals, colors=None):
        """Mesh into caller tensors verts / normals (/ colors) f32 [3*cap_tri, 3].  Returns (demand, rc); rc is 0 or
        TSLAM_E_CAPACITY (outputs saturated at cap_tri), anything else raises.  self.stats = (blocks, stamped,
        touched, remeshed)."""
        n = C.c_int64(0)
        st = (C.c_int32 * 4)()
        rc = self.L.tslam_mesh_update(self.h, float(thres), int(cap_tri), capi.tptr(verts), capi.tptr(normals), capi.tptr(colors),
                                      C.byref(n), st, capi.stream_ptr())
        if rc != capi.E_CAPACITY:
            capi.check(rc)
        self.stats = tuple(int(x) for x in st)
        return int(n.value), rc

    def updated_blocks(self):
        """The blocks remeshed by the last update, in pool order: dict(blocks int32 [n,4] (submap, bx, by, bz),
        first_tri int64 [n], n_tri int32 [n], full).  A superset of the blocks whose triangles changed; n_tri 0 means
        the block's mesh is now empty; full = the last update rebuilt everything (drop what was kept)."""
        import torch
        full = C.c_int32(0)
        blk, first, cnt = capi.count_fill(lambda cap, n, blk, first, cnt: self.L.tslam_mesh_updated_blocks(
            self.h, cap, blk, first, cnt, n, C.byref(full), capi.stream_ptr()), ((4,), torch.int32), ((), torch.int64), ((), torch.int32))
        return dict(blocks=blk, first_tri=first, n_tri=cnt, full=bool(full.value))
