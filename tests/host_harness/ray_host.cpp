// Test-only: compiles the ray-casting header (mujoco_warp_b200/csrc/mjb_ray.cuh) as plain host C++, so that the device source of
// every per-geom ray routine, the geom filters and the closest-hit scan of k_ray runs on the CPU against the reference-generated
// fixture (tests/golden/ray_vectors.npz).  Nothing in the product path uses this file.
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

// k_ray's loop for every (world, ray) pair, one pair at a time (the mesh path through ray_mesh: box test, then the triangles)
extern "C" void hray_rays(int ngeom, int nmesh, int nmeshface, const int* geom_type, const int* geom_bodyid, const int* body_weldid, const int* geom_group,
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
    const v3 p = ld3(pnt + 3 * src), v = ld3(vec + 3 * src);
    float best = MJ_MAXVAL;
    int best_g = -1;
    v3 best_n = ray_zero3();
    for (int g = 0; g < ngeom; g++) {
      v3 n;
      const float x = ray_world_geom(m, geom_xpos + (size_t)w * ngeom * 3, geom_xmat + (size_t)w * ngeom * 9, g, f, bodyexclude[r], p, v, &n);
      if (x >= 0.f && x < best) { best = x; best_g = g; best_n = n; }
    }
    dist[i] = best_g >= 0 ? best : -1.f;
    geomid[i] = best_g;
    st3(normal + 3 * i, best_n);
  }
}
