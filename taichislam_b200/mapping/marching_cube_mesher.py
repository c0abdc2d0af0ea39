"""MarchingCubeMesher - the reference's class surface (marching_cube_mesher.py:12-193) on the
two-pass CUDA marching cubes of libtslam.so (tslam_mc_generate2)."""
import ctypes as C

from .. import _capi as capi
from ..mesh_handle import MeshCache
from .field import Field


class MarchingCubeMesher:
    def __init__(self, mapping, max_triangles=1000000, tsdf_surface_thres=0.1):
        import torch
        self._torch = torch
        dev = torch.device("cuda", torch.cuda.current_device())
        self.max_triangles = max_triangles
        # mesh_vertices pre-filled with -1e6 sentinels (:35-38); colours/normals start at zero like ti fields
        self.mesh_vertices = Field(torch.full((max_triangles * 3, 3), -1000000.0, dtype=torch.float32, device=dev))
        self.mesh_colors = Field(torch.zeros((max_triangles * 3, 3), dtype=torch.float32, device=dev))
        self.mesh_normals = Field(torch.zeros((max_triangles * 3, 3), dtype=torch.float32, device=dev))
        self.mesh_indices = None
        self.num_facelets = Field(torch.zeros(1, dtype=torch.int32, device=dev))
        self.num_vertices = Field(torch.zeros(1, dtype=torch.int32, device=dev))
        self.mapping = mapping
        self.enable_texture = mapping.enable_texture
        self.tsdf_surface_thres = tsdf_surface_thres
        self._cache = None  # incremental mesh of the step-1 calls (mesh_handle.MeshCache)

    def generate_mesh(self, step=1):
        """:192-193 -> generate_mesh_kernel (:180-187).  num_facelets holds the triangle DEMAND; when it exceeds
        max_triangles the buffers hold the first max_triangles (the reference writes out of bounds there, :175-177).
        step 1 goes through the map's incremental mesh, which remeshes only the blocks changed since the previous call
        (the output equals tslam_mc_generate2 bit for bit); other steps take the generic path and drop the cache."""
        m = self.mapping
        m._flush()
        n = C.c_int64(0)
        colors = capi.tptr(self.mesh_colors.t) if self.enable_texture else None  # add_triangle_color (:104-108, :120-125)
        if int(step) == 1:
            if self._cache is None or self._cache.map is not m._h:
                self._drop_cache()
                self._cache = MeshCache(m._h)
            demand, _ = self._cache.update_into(self.tsdf_surface_thres, self.max_triangles, self.mesh_vertices.t,
                                                self.mesh_normals.t, self.mesh_colors.t if self.enable_texture else None)
            n.value = demand
        else:
            self._drop_cache()
            rc = m._h.L.tslam_mc_generate2(m._h.h, int(step), float(self.tsdf_surface_thres), self.max_triangles,
                                           capi.tptr(self.mesh_vertices.t), capi.tptr(self.mesh_normals.t), colors, C.byref(n),
                                           capi.stream_ptr())
            if rc != capi.E_CAPACITY:
                capi.check(rc)
        self.num_facelets[None] = int(n.value)
        # the reference never writes num_vertices (:22) although the node reads it (taichislam_node.py:342)
        self.num_vertices[None] = 3 * min(int(n.value), self.max_triangles)
        print("Total triangles", int(n.value))

    def updated_blocks(self):
        """The blocks the last step-1 generate_mesh remeshed (MeshCache.updated_blocks): where the mesh may have changed."""
        if self._cache is None:
            raise RuntimeError("updated_blocks: no step-1 generate_mesh since the cache was created or dropped")
        return self._cache.updated_blocks()

    def _drop_cache(self):
        if self._cache is not None:
            self._cache.close()
            self._cache = None

    def vertice_num(self):  # :189-190
        return self.num_facelets[None] * 3
