// k_sensor_rangefinder.cu -- rangefinder sensors: the distance along each rangefinder site's z axis to the closest geom.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): sensor.py:810-843 sensor_pos's rangefinder block (:179 _sensor_rangefinder_init,
// then ray.py:1219 rays with no group filter, static geoms included and the site's body excluded) and :568 its _write_scalar.  One
// thread per (world, rangefinder) pair of the launch's world range, flattened world-major as in k_ray, so the lanes of a warp share a
// world and read its geom poses as broadcast loads.  The closest-hit scan is k_ray's (mjb_ray.cuh ray_scan); the distance goes straight
// to the sensor's slot through the cutoff rule of k_sensor, so the launch allocates nothing and stays graph-capturable.
#include "mjb_launch.cuh"
#include "mjb_ray.cuh"

namespace {

constexpr int kRangefinderBlock = 128;

// MESH: the model has meshes; BAT: batched model fields (geom_size / geom_rgba / mat_rgba entry of the world)
template <bool MESH, bool BAT>
__global__ void __launch_bounds__(kRangefinderBlock)
k_sensor_rangefinder(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const __grid_constant__ RangefinderDev rf) {
  const int nrf = rf.nrangefinder;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  // lanes past the last pair stay in the scan (inactive) so that the warp-wide vote of the mesh path sees every lane
  const bool live = i < d.wn * nrf;
  const int k = live ? i / nrf : 0, r = live ? i - k * nrf : 0, w = d.w0 + k;
  MJB_WORLD_MODEL(w)
  const int s = rf.sensor_rangefinder_adr[r], site = m.sensor_objid[s];
  const size_t wb = (size_t)w;
  // sensor.py:179-197: origin at the site, direction along its z axis (column 2 of site_xmat)
  const float* xmat = d.site_xmat + (wb * m.nsite + site) * 9;
  const v3 p = ld3(d.site_xpos + (wb * m.nsite + site) * 3), v = mk3(xmat[2], xmat[5], xmat[8]);
  RayFilter filter;
  for (int g = 0; g < 6; g++) filter.geomgroup[g] = -1;
  filter.flg_static = 1;
  int geomid;
  v3 normal;
  float x = ray_scan<MESH>(m, d.geom_xpos + wb * m.ngeom * 3, d.geom_xmat + wb * m.ngeom * 9, filter, rf.sensor_rangefinder_bodyid[r], live, p, v, &geomid, &normal);
  if (!live) return;
  // sensor.py:57-81 _write_scalar, as k_sensor: cutoff clamps REAL data to [-c, c] and POSITIVE data from above (a miss, -1, stays)
  const float cutoff = m.sensor_cutoff[s];
  const int dt = m.sensor_datatype[s];
  if (cutoff > 0.f) { if (dt == 0) x = fminf(fmaxf(x, -cutoff), cutoff); else if (dt == 1) x = fminf(x, cutoff); }
  d.sensordata[wb * m.nsensordata + m.sensor_adr[s]] = x;
}

}  // namespace

cudaError_t launch_sensor_rangefinder(const ModelDev& m, const DataDev& d, const RangefinderDev& r, cudaStream_t s) {
  const int n = d.wn * r.nrangefinder;  // make_data rejects nworld * nrangefinder past INT_MAX
  if (n <= 0) return cudaSuccess;
  const unsigned grid = (unsigned)((n + kRangefinderBlock - 1) / kRangefinderBlock);
  auto kern = m.nmesh > 0 ? (m.batched ? k_sensor_rangefinder<true, true> : k_sensor_rangefinder<true, false>)
                          : (m.batched ? k_sensor_rangefinder<false, true> : k_sensor_rangefinder<false, false>);
  return launch(kern, grid, kRangefinderBlock, 0, s, m, d, r);
}
