// Test-only: compiles the closest-hit scan the ray and rangefinder kernels share (mujoco_warp_b200/csrc/mjb_ray.cuh ray_scan) as plain host
// C++, one ray at a time (each ray is its own warp, so the mesh path's warp vote is the ray's own box test).  Same signature as
// ray_host.cpp's hray_rays, so that tests/test_ray_vectors.py's `cast` drives it.  Nothing in the product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <algorithm>
using std::max;
using std::min;
// warp intrinsics mjb_math.cuh's helpers name (unused by the ray routines)
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
#include "../../mujoco_warp_b200/csrc/mjb_ray.cuh"

extern "C" void hrf_scan(int ngeom, int nmesh, int nmeshface, const int* geom_type, const int* geom_bodyid, const int* body_weldid, const int* geom_group,
                         const int* geom_matid, const int* geom_dataid, const float* geom_size, const float* geom_rgba, const float* mat_rgba,
                         const int* mesh_vertadr, const int* mesh_faceadr, const int* mesh_face, const float* mesh_vert, int nworld, const float* geom_xpos,
                         const float* geom_xmat, int nray, int pnt_nbatch, const float* pnt, const float* vec, const int* geomgroup, int flg_static,
                         const int* bodyexclude, float* dist, int* geomid, float* normal) {
  ModelDev m;
  memset(&m, 0, sizeof m);
  m.ngeom = ngeom; m.nmesh = nmesh; m.nmeshface = nmeshface;
  m.geom_type = geom_type; m.geom_bodyid = geom_bodyid; m.body_weldid = body_weldid; m.geom_group = geom_group; m.geom_matid = geom_matid;
  m.geom_dataid = geom_dataid; m.geom_size = geom_size; m.geom_rgba = geom_rgba; m.mat_rgba = mat_rgba;
  m.mesh_vertadr = mesh_vertadr; m.mesh_faceadr = mesh_faceadr; m.mesh_face = mesh_face; m.mesh_vert = mesh_vert;
  RayFilter f;
  for (int k = 0; k < 6; k++) f.geomgroup[k] = geomgroup[k];
  f.flg_static = flg_static != 0;
  for (long i = 0; i < (long)nworld * nray; i++) {
    const int w = (int)(i / nray), r = (int)(i % nray);
    const long src = (long)(pnt_nbatch == 1 ? 0 : w) * nray + r;
    v3 n;
    dist[i] = ray_scan<true>(m, geom_xpos + (size_t)w * ngeom * 3, geom_xmat + (size_t)w * ngeom * 9, f, bodyexclude[r], true, ld3(pnt + 3 * src),
                             ld3(vec + 3 * src), geomid + i, &n);
    st3(normal + 3 * i, n);
  }
}
