// k_sensor_collision.cu -- distance / normal / fromto sensors, one warp per world (mjb_sensor_collision.cuh).
//
// Lanes take the world's unique sensor geom pairs (a pair shared by several sensors runs once), each pair's first least-distance contact
// goes to shared memory, then lanes take the sensors and reduce over their pairs in the reference's loop order.  The kernel writes only
// the collision sensors' slots of sensordata (k_sensor skips them), and only in the CCD_MESH build of the convex code, so that one
// instance serves models with and without mesh geoms.  k_sensor_collision_large.cu builds the same source with CCD_MESH = 2.
#ifndef CCD_MESH
#define CCD_MESH 1
#endif
#include "mjb_launch.cuh"
#include "mjb_sensor_collision.cuh"
#include "mjb_types.cuh"

namespace {

#if CCD_MESH == 2
#define SC_KERNEL k_sensor_collision_large
#define SC_EXTRA_PARAM , const __grid_constant__ MeshClipDev clipdev
#else
#define SC_KERNEL k_sensor_collision
#define SC_EXTRA_PARAM
#endif

template <bool BAT>
__global__ void __launch_bounds__(32)
SC_KERNEL(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const __grid_constant__ SensorCollisionDev c SC_EXTRA_PARAM) {
  extern __shared__ float smem[];  // nsensorcollision x SC_WORDS pair results, then the EPA scratch slots
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  const int sw = ccd_scratch_words(c.sensor_collision_epa_iterations);
  float* slots = smem + SC_WORDS * c.nsensorcollision;
  const float *gxpos = d.geom_xpos + wb * 3 * m.ngeom, *gxmat = d.geom_xmat + wb * 9 * m.ngeom;
  bool ovf = false;
  for (int p = lane; p < c.nsensorcollision; p += 32) {
    const int* pr = c.sensor_collision_pair + SC_PAIR_WORDS * p;
    // a GJK / EPA pair's slot: its rank among those pairs when there are at most 32 (pairs of one pass have distinct ranks), else the lane's
    float* scratch = pr[3] < 0 ? nullptr : slots + (size_t)(c.nsensorcollision_ccd <= 32 ? pr[3] : lane) * sw;
#if CCD_MESH == 2
    // the multi-contact scratch has the same slots, nslot >= min(32, nsensorcollision_ccd) of them
    const int slot = pr[3] < 0 ? 0 : (c.nsensorcollision_ccd <= 32 ? pr[3] : lane);
    const CcdClip mc = {clipdev.scratch + ((size_t)w * clipdev.nslot + slot) * mesh_clip_words(clipdev), mesh_clip_poly(clipdev), mesh_clip_deg(clipdev)};
#endif
    ovf |= sensor_pair(m, gxpos, gxmat, pr[0], pr[1], pr[2], c.sensor_collision_epa_iterations, scratch, smem + SC_WORDS * p CCD_CLIP_ARG);
  }
  if (__any_sync(FULL_MASK, ovf) && lane == 0) d.overflow[w] |= OVF_EPA_HORIZON;  // k_collision, earlier in the stream, wrote its bits
  __syncwarp();
  float* out = d.sensordata + wb * m.nsensordata;
  for (int i = lane; i < c.nsensorcollision_sensor; i += 32) sensor_collision_reduce(m, c, i, smem, out);
}

}  // namespace

#if CCD_MESH == 2
cudaError_t launch_sensor_collision_large(const ModelDev& m, const DataDev& d, const SensorCollisionDev& c, const MeshClipDev& mc, cudaStream_t s) {
  return launch(m.batched ? k_sensor_collision_large<true> : k_sensor_collision_large<false>, d.wn, 32, smem_sensor_collision(c), s, m, d, c, mc);
}
#else
size_t smem_sensor_collision(const SensorCollisionDev& c) {
  const int nslot = c.nsensorcollision_ccd < 32 ? c.nsensorcollision_ccd : 32;
  return sizeof(float) * ((size_t)SC_WORDS * c.nsensorcollision + (size_t)nslot * ccd_scratch_words(c.sensor_collision_epa_iterations));
}

cudaError_t launch_sensor_collision(const ModelDev& m, const DataDev& d, const SensorCollisionDev& c, cudaStream_t s) {
  return launch(m.batched ? k_sensor_collision<true> : k_sensor_collision<false>, d.wn, 32, smem_sensor_collision(c), s, m, d, c);
}
#endif
