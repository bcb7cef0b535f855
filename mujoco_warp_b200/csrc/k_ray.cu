// k_ray.cu -- ray casting: the closest geom every ray of every world hits.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): ray.py:1219 rays / :907 _ray without a render context (no BVH).
// One thread per (world, ray) pair, flattened world-major (i = w * nray + r), so the three outputs are written coalesced.  Every
// thread scans the geoms in ascending order (mjb_ray.cuh ray_scan, shared with the rangefinder sensor): the loop index is
// warp-uniform, so the geom-type switch and the model-constant loads do not diverge, and the lanes of one world read the same
// geom_xpos / geom_xmat address (one broadcast load).  The closest hit is replaced only on a strictly smaller distance, so ties go
// to the lowest geom id, as the reference's argmin within a tile and strict compare across tiles do (ray.py:994-1004); a ray's
// result does not depend on scheduling.
#include "mjb_launch.cuh"
#include "mjb_ray.cuh"

namespace {

constexpr int kRayBlock = 128;

// MESH: the model has meshes (the triangle path is compiled in); BAT: batched model fields (geom_size / geom_rgba / mat_rgba
// entry w % nbatch)
template <bool MESH, bool BAT>
__global__ void __launch_bounds__(kRayBlock)
k_ray(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const float* __restrict__ pnt, const float* __restrict__ vec, int nray,
      int pnt_nbatch, const RayFilter filter, const int* __restrict__ bodyexclude, float* __restrict__ dist_out, int* __restrict__ geomid_out,
      float* __restrict__ normal_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  // lanes past the last ray stay in the loop (inactive) so that the warp-wide vote of the mesh path sees every lane
  const bool live = i < d.nworld * nray;
  const int w = live ? i / nray : 0, r = live ? i - w * nray : 0;
  MJB_WORLD_MODEL(w)
  const size_t src = (size_t)(pnt_nbatch == 1 ? 0 : w) * nray + r;
  const v3 p = live ? ld3(pnt + 3 * src) : ray_zero3(), v = live ? ld3(vec + 3 * src) : ray_zero3();
  const int bx = live ? bodyexclude[r] : -1;
  int best_g;
  v3 best_n;
  const float best = ray_scan<MESH>(m, d.geom_xpos + (size_t)w * m.ngeom * 3, d.geom_xmat + (size_t)w * m.ngeom * 9, filter, bx, live, p, v, &best_g, &best_n);
  if (!live) return;
  dist_out[i] = best;
  geomid_out[i] = best_g;
  st3(normal_out + 3 * (size_t)i, best_n);
}

}  // namespace

cudaError_t launch_ray(const ModelDev& m, const DataDev& d, const float* pnt, const float* vec, int nray, int pnt_nbatch, const int* geomgroup, int flg_static,
                       const int* bodyexclude, float* dist, int* geomid, float* normal, cudaStream_t s) {
  const int n = d.nworld * nray;  // the caller rejects sizes past INT_MAX
  if (n <= 0) return cudaSuccess;
  RayFilter f;
  for (int k = 0; k < 6; k++) f.geomgroup[k] = geomgroup ? geomgroup[k] : -1;
  f.flg_static = flg_static != 0;
  const unsigned grid = (unsigned)((n + kRayBlock - 1) / kRayBlock);
  auto kern = m.nmesh > 0 ? (m.batched ? k_ray<true, true> : k_ray<true, false>) : (m.batched ? k_ray<false, true> : k_ray<false, false>);
  return launch(kern, grid, kRayBlock, 0, s, m, d, pnt, vec, nray, pnt_nbatch, f, bodyexclude, dist, geomid, normal);
}
