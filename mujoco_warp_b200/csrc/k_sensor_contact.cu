// k_sensor_contact.cu -- <contact> sensors, one warp per world (mjb_sensor_contact.cuh).
//
// The sensors one after the other, each through one shared-memory buffer of contact_sensor_maxmatch x 3 words (pool index, criterion,
// direction):
//   match   lanes take the world's contacts in pool order, 32 at a time; a ballot prefix appends the matches in pool order, and the match
//           count keeps counting past the buffer (OVF_CONTACT_MATCH once it does)
//   sort    mindist / maxforce: the stored matches by (criterion, pool index)
//   write   lanes take the slots (none / mindist / maxforce: stored match i, or zeros), or the stored matches' netforce sums
// The kernel writes only the contact sensors' slots of sensordata (k_sensor skips them).  Deterministic: no atomics, fixed reduction order.
#include "mjb_launch.cuh"
#include "mjb_sensor_contact.cuh"
#include "mjb_types.cuh"

namespace {

template <bool BAT>
__global__ void __launch_bounds__(32)
k_sensor_contact(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const __grid_constant__ SensorContactDev c) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x, w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const size_t wb = (size_t)w;
  const int maxmatch = c.contact_sensor_maxmatch;
  int* bid = (int*)smem;
  float *bcrit = smem + maxmatch, *bdir = smem + 2 * maxmatch;
  const float* force = d.efc_force + wb * d.njmax;
  float* out = d.sensordata + wb * m.nsensordata;
  const int c0 = d.world_conadr[w], c1 = c0 + d.world_ncon[w];  // already clamped by k_collision to the per-world cap and the pool
  bool ovf = false;
#pragma unroll 1
  for (int k = 0; k < c.nsensorcontact; k++) {
    const int s = c.sensor_contact_adr[k];
    const int dataspec = c.sensor_intprm[3 * s], reduce = c.sensor_intprm[3 * s + 1], num = c.sensor_intprm[3 * s + 2];
    const int otype = m.sensor_objtype[s], oid = m.sensor_objid[s], rtype = m.sensor_reftype[s], rid = m.sensor_refid[s];
    int nmatch = 0;
#pragma unroll 1
    for (int cb = c0; cb < c1; cb += 32) {
      const int ci = cb + lane;
      int dir = 0;
      if (ci < c1 && (d.contact_type[ci] & CONTACT_TYPE_CONSTRAINT)) {
        const v3 cpos = ld3(d.contact_pos + 3 * (size_t)ci);
        if (otype != OBJ_SITE || contact_inside_site(ld3(d.site_xpos + (wb * m.nsite + oid) * 3), d.site_xmat + (wb * m.nsite + oid) * 9, ld3(m.site_size + 3 * oid),
                                                     m.site_type[oid], cpos)) {
          const int g1 = d.contact_geom[2 * (size_t)ci], g2 = d.contact_geom[2 * (size_t)ci + 1];
          dir = contact_match_dir(m.body_parentid, otype, oid, rtype, rid, g1, m.geom_bodyid[g1], g2, m.geom_bodyid[g2]);
        }
      }
      const unsigned ballot = __ballot_sync(FULL_MASK, dir != 0);
      const int slot = nmatch + __popc(ballot & ((1u << lane) - 1u));
      if (dir != 0 && slot < maxmatch) {
        float crit = 0.f;
        if (reduce == CSR_MINDIST) crit = d.contact_dist[ci];
        else if (reduce == CSR_MAXFORCE) {
          float f[6];
          contact_force_decode(m.cone, d.njmax, force, d.contact_efc_address + (size_t)ci * m.nmaxpyramid, d.contact_friction + 5 * (size_t)ci, d.contact_dim[ci], f);
          crit = -(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
        }
        bid[slot] = ci; bcrit[slot] = crit; bdir[slot] = (float)dir;
      }
      nmatch += __popc(ballot);
    }
    ovf |= nmatch > maxmatch;
    const int nstore = min(nmatch, maxmatch);
    __syncwarp();
    if ((reduce == CSR_MINDIST || reduce == CSR_MAXFORCE) && nstore > 1) contact_sort(bid, bcrit, bdir, nstore, lane, 32, [] { __syncwarp(); });
    const int adr = m.sensor_adr[s], size = contact_slot_size(dataspec);
    if (reduce == CSR_NETFORCE) {
      float acc[CNF_WORDS] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int i = lane; i < nstore; i += 32) {
        const int ci = bid[i];
        float f[6];
        contact_force_decode(m.cone, d.njmax, force, d.contact_efc_address + (size_t)ci * m.nmaxpyramid, d.contact_friction + 5 * (size_t)ci, d.contact_dim[ci], f);
        contact_netforce_add(bdir[i], f, d.contact_pos + 3 * (size_t)ci, d.contact_frame + 9 * (size_t)ci, acc);
      }
      for (int j = 0; j < CNF_WORDS; j++) acc[j] = warp_sum(acc[j]);
      if (lane == 0) contact_netforce_write(dataspec, nmatch, acc, out + adr);
      for (int i = size + lane; i < num * size; i += 32) out[adr + i] = 0.f;  // slots 2..num
    } else {
      const int nslot = min(nstore, num);
      for (int i = lane; i < num; i += 32) {
        float* o = out + adr + i * size;
        if (i < nslot) {
          const int ci = bid[i];
          float f[6];
          contact_force_decode(m.cone, d.njmax, force, d.contact_efc_address + (size_t)ci * m.nmaxpyramid, d.contact_friction + 5 * (size_t)ci, d.contact_dim[ci], f);
          contact_slot_write(dataspec, nmatch, bdir[i], f, d.contact_dist[ci], d.contact_pos + 3 * (size_t)ci, d.contact_frame + 9 * (size_t)ci, o);
        } else {
          for (int j = 0; j < size; j++) o[j] = 0.f;
        }
      }
    }
    __syncwarp();  // the next sensor reuses the buffer
  }
  if (ovf && lane == 0) d.overflow[w] |= OVF_CONTACT_MATCH;  // k_collision, earlier in the stream, wrote its bits
}

}  // namespace

size_t smem_sensor_contact(const SensorContactDev& c) { return sizeof(float) * 3 * (size_t)c.contact_sensor_maxmatch; }

cudaError_t launch_sensor_contact(const ModelDev& m, const DataDev& d, const SensorContactDev& c, cudaStream_t s) {
  return launch(m.batched ? k_sensor_contact<true> : k_sensor_contact<false>, d.wn, 32, smem_sensor_contact(c), s, m, d, c);
}
