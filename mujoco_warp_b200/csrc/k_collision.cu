// k_collision.cu -- fused collision stage: NXN broadphase + primitive narrowphase + contact write.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): collision_driver.py:684-770 (_nxn_broadphase: one thread
// per (world, pair), one global atomic per surviving pair), :98-334 (plane/sphere/AABB/OBB filters),
// collision_primitive.py:1352-1513 (_primitive_narrowphase: naconmax threads, most idle), collision_primitive_core.py:47-302
// (plane-sphere, sphere-sphere, sphere-capsule, capsule-capsule, plane-capsule), :305-1433 (ellipsoid / cylinder / box pairs,
// mjb_colliders.cuh; only in the k_collision<8> instantiation, chosen when the model has such geoms),
// collision_core.py:213-470 (write_contact, contact parameter mixing).
//
// Design: one warp owns one world.  Lanes test the model's precomputed pair list, survivors are compacted with
// ballot/popc in pair order, narrowphase runs densely on the compacted list, contacts are staged in shared memory and the
// world claims ONE contiguous block of the global contact pool with a single atomicAdd (the reference issues one atomic
// per pair and one per contact).  Within a world the contact order is deterministic (pair order, then contact index);
// only the position of a world's block inside the pool depends on scheduling.  Data.contact keeps the reference's global
// pool layout (types.py:1975-2018) so [0, nacon) is densely packed.
#include "mjb_ccd.cuh"
#include "mjb_colliders.cuh"
#include <cstdlib>

#include "mjb_math.cuh"
#include "mjb_team.cuh"
#include "mjb_types.cuh"

namespace {

constexpr int STAGE_WORDS = 13;  // dist, pos[3], frame[9]

__host__ __device__ inline int world_con_cap(const DataDev& d) { return 2 * d.nconmax > 32 ? 2 * d.nconmax : 32; }
__host__ __device__ inline int surv_cap(const ModelDev& m) { return m.nxn_npair < 1024 ? m.nxn_npair : 1024; }

constexpr int CCD_LANES = 4;  // geom pairs that run GJK / EPA concurrently in one warp (each needs a polytope in shared memory)

struct ColLayout { int gxpos, gxmat, surv, stage, sgeom, ccd, sap, bar, total; };
__host__ __device__ inline ColLayout col_layout(const ModelDev& m, const DataDev& d) {
  ColLayout L;
  int o = 0;
  auto take = [&](int n) { int r = o; o += n; return r; };
  // geom poses first, each on a 16-byte boundary: staged with one bulk-async copy apiece when the world's rows are aligned in global memory
  L.gxpos = take((3 * m.ngeom + 3) & ~3); L.gxmat = take((9 * m.ngeom + 3) & ~3);
  L.surv = take(surv_cap(m));
  L.stage = take(STAGE_WORDS * world_con_cap(d));
  L.sgeom = take(4 * world_con_cap(d));  // g1, g2, geomcollisionid, pairid
  L.ccd = take(m.has_convex_pair ? CCD_LANES * ccd_scratch_words(m.epa_iterations) : 0);
  L.sap = take(m.broadphase != 0 ? 4 * m.ngeom : 0);  // sweep-and-prune: projection bounds, sorted lower bounds, ranks
  o = (o + 3) & ~3;
  L.bar = take(4);  // mbarrier of the staging copies (8 bytes in a 16-byte slot)
  L.total = (o + 3) & ~3;
  return L;
}

__device__ __forceinline__ bool plane_filter(float size1, float size2, float margin1, float margin2, v3 xp1, v3 xp2, const float* xm1, const float* xm2) {
  if (size1 == 0.f) return dot(xp2 - xp1, matcol(xm1, 2)) <= size2 + margin1 + margin2;
  if (size2 == 0.f) return dot(xp1 - xp2, matcol(xm2, 2)) <= size1 + margin1 + margin2;
  return true;
}
__device__ __forceinline__ bool sphere_filter(float size1, float size2, float margin1, float margin2, v3 xp1, v3 xp2) {
  const float bound = size1 + size2 + margin1 + margin2;
  const v3 dif = xp2 - xp1;
  return dot(dif, dif) <= bound * bound;
}
__device__ bool aabb_filter(v3 c1, v3 c2, v3 s1, v3 s2, float margin, v3 xp1, v3 xp2, const float* xm1, const float* xm2) {
  const v3 ce1 = matvec(xm1, c1) + xp1, ce2 = matvec(xm2, c2) + xp2;
  // extent of a rotated box along world axis a = sum_k |R[a][k]| * size[k]  (max over the 8 corners)
  const float e1x = fabsf(xm1[0]) * s1.x + fabsf(xm1[1]) * s1.y + fabsf(xm1[2]) * s1.z;
  const float e1y = fabsf(xm1[3]) * s1.x + fabsf(xm1[4]) * s1.y + fabsf(xm1[5]) * s1.z;
  const float e1z = fabsf(xm1[6]) * s1.x + fabsf(xm1[7]) * s1.y + fabsf(xm1[8]) * s1.z;
  const float e2x = fabsf(xm2[0]) * s2.x + fabsf(xm2[1]) * s2.y + fabsf(xm2[2]) * s2.z;
  const float e2y = fabsf(xm2[3]) * s2.x + fabsf(xm2[4]) * s2.y + fabsf(xm2[5]) * s2.z;
  const float e2z = fabsf(xm2[6]) * s2.x + fabsf(xm2[7]) * s2.y + fabsf(xm2[8]) * s2.z;
  if (ce1.x + e1x + margin < ce2.x - e2x || ce2.x + e2x + margin < ce1.x - e1x) return false;
  if (ce1.y + e1y + margin < ce2.y - e2y || ce2.y + e2y + margin < ce1.y - e1y) return false;
  if (ce1.z + e1z + margin < ce2.z - e2z || ce2.z + e2z + margin < ce1.z - e1z) return false;
  return true;
}
__device__ bool obb_filter(v3 c1, v3 c2, v3 s1, v3 s2, float margin, v3 xp1, v3 xp2, const float* xm1, const float* xm2) {
  const v3 xc1 = matvec(xm1, c1) + xp1, xc2 = matvec(xm2, c2) + xp2;
  v3 n[6];
  for (int k = 0; k < 3; k++) { n[k] = matcol(xm1, k); n[3 + k] = matcol(xm2, k); }
  for (int a = 0; a < 6; a++) {
    const float p0 = dot(xc1, n[a]), p1 = dot(xc2, n[a]);
    const float r0 = fabsf(s1.x * dot(n[0], n[a])) + fabsf(s1.y * dot(n[1], n[a])) + fabsf(s1.z * dot(n[2], n[a]));
    const float r1 = fabsf(s2.x * dot(n[3], n[a])) + fabsf(s2.y * dot(n[4], n[a])) + fabsf(s2.z * dot(n[5], n[a]));
    if (r0 + r1 + margin < fabsf(p1 - p0)) return false;
  }
  return true;
}

__device__ __forceinline__ float plane_sphere(v3 n, v3 ppos, v3 spos, float r, v3* pos) {
  const float dist = dot(spos - ppos, n) - r;
  *pos = spos - n * (r + 0.5f * dist);
  return dist;
}
__device__ __forceinline__ float sphere_sphere(v3 pos1, float r1, v3 pos2, float r2, v3* pos, v3* n) {
  const v3 dir = pos2 - pos1;
  float dist = length(dir);
  *n = dist == 0.f ? mk3(1.f, 0.f, 0.f) : dir * (1.0f / dist);
  dist = dist - (r1 + r2);
  *pos = pos1 + (*n) * (r1 + 0.5f * dist);
  return dist;
}

struct ConParams { float margin, gap; int condim; float friction[5], solref[2], solreffriction[2], solimp[5]; };

// collision_core.py:294-412 for geom pairs (pairid == -1)
__device__ void contact_params(const ModelDev& m, int g1, int g2, int pairid, ConParams* p) {
  if (pairid > -1) {  // explicit <pair>: every parameter comes from the pair (collision_core.py:305-307, 343-349)
    p->margin = m.pair_margin[pairid]; p->gap = m.pair_gap[pairid]; p->condim = m.pair_dim[pairid];
    for (int i = 0; i < 5; i++) { p->friction[i] = fmaxf(MJ_MINMU, m.pair_friction[5 * pairid + i]); p->solimp[i] = m.pair_solimp[5 * pairid + i]; }
    for (int i = 0; i < 2; i++) { p->solref[i] = m.pair_solref[2 * pairid + i]; p->solreffriction[i] = m.pair_solreffriction[2 * pairid + i]; }
    return;
  }
  p->solreffriction[0] = 0.f; p->solreffriction[1] = 0.f;
  p->margin = m.geom_margin[g1] + m.geom_margin[g2];
  p->gap = m.geom_gap[g1] + m.geom_gap[g2];
  const float solmix1 = m.geom_solmix[g1], solmix2 = m.geom_solmix[g2];
  const int p1 = m.geom_priority[g1], p2 = m.geom_priority[g2];
  float mix, f0, f1, f2;
  if (p1 > p2) {
    mix = 1.f; p->condim = m.geom_condim[g1];
    f0 = m.geom_friction[3 * g1]; f1 = m.geom_friction[3 * g1 + 1]; f2 = m.geom_friction[3 * g1 + 2];
  } else if (p2 > p1) {
    mix = 0.f; p->condim = m.geom_condim[g2];
    f0 = m.geom_friction[3 * g2]; f1 = m.geom_friction[3 * g2 + 1]; f2 = m.geom_friction[3 * g2 + 2];
  } else {
    mix = safe_div(solmix1, solmix1 + solmix2);
    if (solmix1 < MJ_MINVAL && solmix2 < MJ_MINVAL) mix = 0.5f;
    if (solmix1 < MJ_MINVAL && solmix2 >= MJ_MINVAL) mix = 0.f;
    if (solmix1 >= MJ_MINVAL && solmix2 < MJ_MINVAL) mix = 1.f;
    p->condim = max(m.geom_condim[g1], m.geom_condim[g2]);
    f0 = fmaxf(m.geom_friction[3 * g1], m.geom_friction[3 * g2]);
    f1 = fmaxf(m.geom_friction[3 * g1 + 1], m.geom_friction[3 * g2 + 1]);
    f2 = fmaxf(m.geom_friction[3 * g1 + 2], m.geom_friction[3 * g2 + 2]);
  }
  p->friction[0] = fmaxf(MJ_MINMU, f0); p->friction[1] = fmaxf(MJ_MINMU, f0); p->friction[2] = fmaxf(MJ_MINMU, f1);
  p->friction[3] = fmaxf(MJ_MINMU, f2); p->friction[4] = fmaxf(MJ_MINMU, f2);
  const float *sr1 = m.geom_solref + 2 * g1, *sr2 = m.geom_solref + 2 * g2;
  if (sr1[0] > 0.f && sr2[0] > 0.f) { p->solref[0] = mix * sr1[0] + (1.f - mix) * sr2[0]; p->solref[1] = mix * sr1[1] + (1.f - mix) * sr2[1]; }
  else { p->solref[0] = fminf(sr1[0], sr2[0]); p->solref[1] = fminf(sr1[1], sr2[1]); }
  p->solreffriction[0] = p->solreffriction[1] = 0.f;
  for (int i = 0; i < 5; i++) p->solimp[i] = mix * m.geom_solimp[5 * g1 + i] + (1.f - mix) * m.geom_solimp[5 * g2 + i];
}

#if CCD_MESH
// collision_core.py:60-140 geom(): a mesh geom carries its asset's vertex block, hull graph and hull polygon tables
__device__ __forceinline__ void fill_mesh(const ModelDev& m, int g, CGeom& c) {
  c.index = -1; c.vertnum = 0; c.polynum = 0; c.vert = nullptr; c.polynormal = nullptr; c.graph = nullptr;
  c.polyvertadr = c.polyvertnum = c.polyvert = c.polymapadr = c.polymapnum = c.polymap = nullptr;
  if (c.type != GEOM_MESH) return;
  const int id = m.geom_dataid[g];
  if (id < 0) return;
  const int vadr = m.mesh_vertadr[id], padr = m.mesh_polyadr[id];
  c.vert = m.mesh_vert + 3 * vadr; c.vertnum = m.mesh_vertnum[id];
  c.graph = m.mesh_graphadr[id] >= 0 ? m.mesh_graph + m.mesh_graphadr[id] : nullptr;
  c.polynum = m.mesh_polynum[id]; c.polynormal = m.mesh_polynormal + 3 * padr;
  c.polyvertadr = m.mesh_polyvertadr + padr; c.polyvertnum = m.mesh_polyvertnum + padr; c.polyvert = m.mesh_polyvert;
  c.polymapadr = m.mesh_polymapadr + vadr; c.polymapnum = m.mesh_polymapnum + vadr; c.polymap = m.mesh_polymap;
}
#endif

// MAXC = contacts one geom pair can produce: 2 for plane/sphere/capsule-only models (everything stays in registers),
// 8 once boxes, cylinders or ellipsoids are present.
template <int MAXC, bool BAT>
__global__ void __launch_bounds__(64, MAXC == 2 ? 16 : 8)
k_collision(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;  // every warp of the block owns one world (its own shared-memory slice)
  const int w = blockIdx.x * (blockDim.x >> 5) + warp + d.w0;
  if (w >= d.nworld || w >= d.w0 + d.wn) return;
  MJB_WORLD_MODEL(w)
  const ColLayout L = col_layout(mp, d);
  float* S = smem + warp * L.total;
  float *gxpos = S + L.gxpos, *gxmat = S + L.gxmat, *stage = S + L.stage;
  int *surv = (int*)(S + L.surv), *sgeom = (int*)(S + L.sgeom);
  const int ng = m.ngeom, scap = surv_cap(m), ccap = world_con_cap(d);
  const size_t wb = (size_t)w;

  if (d.nconmax == 0 || (m.disableflags & (DSBL_CONSTRAINT | DSBL_CONTACT))) {
    if (lane == 0) { d.world_conadr[w] = 0; d.world_ncon[w] = 0; }
    return;
  }
  {  // cp.async.bulk (SASS UBLKCP) when both rows are 16-byte aligned (ngeom a multiple of 4), a lane loop otherwise
    Stager st;
    st.init(reinterpret_cast<uint64_t*>(S + L.bar), lane);
    st.load(gxpos, d.geom_xpos + wb * 3 * ng, 3 * ng);
    st.load(gxmat, d.geom_xmat + wb * 9 * ng, 9 * ng);
    st.load_wait();
  }

  // ---- sweep-and-prune option (collision_driver.py:582-682): bounding-sphere projections on the reference's fixed axis, each
  // geom's position in the sort by lower bound.  A pair is a sweep candidate when every geom sorted between the two starts
  // below the earlier geom's upper bound (the reference's range also takes in the first neighbour past it,
  // collision_core.py:516-519); candidates then go through the same filters.  Survivors keep pair-list order here (the
  // reference's own order comes out of atomics).
  float *sap_lo = S + L.sap, *sap_hi = sap_lo + ng, *sap_sorted = sap_hi + ng;
  int* sap_rank = (int*)(sap_sorted + ng);
  const bool sap = m.broadphase != 0;
  if (sap) {
    const v3 dir = normalize(mk3(0.5935f, 0.7790f, 0.1235f));
    for (int g = lane; g < ng; g += 32) {
      float rb = m.geom_rbound[g];
      if (rb == 0.f) rb = MJ_MAXVAL;
      const float radius = rb + m.geom_margin[g] + m.geom_gap[g], center = dot(dir, ld3(gxpos + 3 * g));
      const bool ok = center == center;
      sap_lo[g] = ok ? center - radius : MJ_MAXVAL; sap_hi[g] = ok ? center + radius : MJ_MAXVAL;
    }
    __syncwarp();
    for (int g = lane; g < ng; g += 32) {
      const float lo = sap_lo[g];
      int r = 0;
      for (int h = 0; h < ng; h++) { const float lh = sap_lo[h]; r += (lh < lo || (lh == lo && h < g)) ? 1 : 0; }
      sap_rank[g] = r; sap_sorted[r] = lo;
    }
    __syncwarp();
  }

  // ---- broadphase: lanes over the filtered pair list, ordered compaction of survivors
  int nsurv = 0, ntotal = 0;
#pragma unroll 1
  for (int e0 = 0; e0 < m.nxn_npair; e0 += 32) {
    const int e = e0 + lane;
    bool pass = false;
    if (e < m.nxn_npair) {
      const int g1 = m.nxn_geom_pair[2 * e], g2 = m.nxn_geom_pair[2 * e + 1];
      const float rb1 = m.geom_rbound[g1], rb2 = m.geom_rbound[g2];
      const float em1 = m.geom_margin[g1] + m.geom_gap[g1], em2 = m.geom_margin[g2] + m.geom_gap[g2];
      const v3 xp1 = ld3(gxpos + 3 * g1), xp2 = ld3(gxpos + 3 * g2);
      const float *xm1 = gxmat + 9 * g1, *xm2 = gxmat + 9 * g2;
      pass = true;
      if (rb1 == 0.f || rb2 == 0.f) {
        if (m.broadphase_filter & BF_PLANE) pass = plane_filter(rb1, rb2, em1, em2, xp1, xp2, xm1, xm2);
      } else {
        if ((m.broadphase_filter & BF_SPHERE) && !sphere_filter(rb1, rb2, em1, em2, xp1, xp2)) pass = false;
        if (pass && (m.broadphase_filter & (BF_AABB | BF_OBB))) {
          const v3 c1 = ld3(m.geom_aabb + 6 * g1), s1 = ld3(m.geom_aabb + 6 * g1 + 3), c2 = ld3(m.geom_aabb + 6 * g2), s2 = ld3(m.geom_aabb + 6 * g2 + 3);
          if ((m.broadphase_filter & BF_AABB) && !aabb_filter(c1, c2, s1, s2, em1 + em2, xp1, xp2, xm1, xm2)) pass = false;
          if (pass && (m.broadphase_filter & BF_OBB) && !obb_filter(c1, c2, s1, s2, em1 + em2, xp1, xp2, xm1, xm2)) pass = false;
        }
      }
      pass = pass || m.nxn_pairid[2 * e + 1] >= 0;
      if (sap) {
        const int ra = sap_rank[g1], rb_ = sap_rank[g2], ri = min(ra, rb_), rj = max(ra, rb_);
        pass = pass && (rj == ri + 1 || sap_sorted[rj - 1] <= sap_hi[ra < rb_ ? g1 : g2]);
      }
    }
    const unsigned bal = __ballot_sync(FULL_MASK, pass);
    ntotal += __popc(bal);
    // sensor-only pairs (pairid[0] == -2) are counted but produce no constraint contact
    const bool keep = pass && m.nxn_pairid[2 * e] != -2;
    const unsigned kb = __ballot_sync(FULL_MASK, keep);
    if (keep) {
      const int pos = nsurv + __popc(kb & ((1u << lane) - 1u));
      if (pos < scap) surv[pos] = e;
    }
    nsurv += __popc(kb);
  }
  int ovf = 0;
  if (nsurv > scap) { nsurv = scap; ovf |= OVF_BROADPHASE; }
  __syncwarp();

  // ---- narrowphase on the compacted list; contacts staged in shared memory.  Order inside a world: convex (GJK / EPA) pairs
  // first, by pair type in the reference's table order, then primitive pairs (the order the reference produces when its
  // launches run sequentially: collision_driver.py:877, collision_convex.py:1369); within a type, pair-list order.
  int ncon = 0;
  if (MAXC >= 8 && m.has_convex_pair) {
    float* ccd_scratch = S + L.ccd;
    const int sw = ccd_scratch_words(m.epa_iterations);
    const bool nativeccd = !(m.disableflags & DSBL_NATIVECCD);
#pragma unroll 1
    for (int rank = 0; rank < CCD_NRANK; rank++) {
#pragma unroll 1
      for (int s0 = 0; s0 < nsurv; s0 += 32) {
        const int si = s0 + lane;
        int g1 = 0, g2 = 0, pid = -1;
        bool mine = false;
        if (si < nsurv) {
          const int e = surv[si];
          g1 = m.nxn_geom_pair[2 * e]; g2 = m.nxn_geom_pair[2 * e + 1];
          if (m.geom_type[g1] > m.geom_type[g2]) { const int t = g1; g1 = g2; g2 = t; }
          mine = convex_rank(m.geom_type[g1], m.geom_type[g2], nativeccd) == rank;
          pid = m.npair > 0 ? m.nxn_pairid[2 * e] : -1;
        }
        unsigned todo = __ballot_sync(FULL_MASK, mine);
        while (todo) {
          unsigned batch = 0, t = todo;
          for (int k = 0; k < CCD_LANES && t; k++) { batch |= t & (0u - t); t &= t - 1; }
          todo &= ~batch;
          const bool active = (batch >> lane) & 1u;
          int nhit = 0;  // contacts of this lane's pair (box pairs recover up to 4)
          float dist = 0.f;
          v3 w1[4], w2[4], nrm = mk3(1.f, 0.f, 0.f);
          if (active) {
            const int slot = __popc(batch & ((1u << lane) - 1u));
            const float margin = pid > -1 ? m.pair_margin[pid] : m.geom_margin[g1] + m.geom_margin[g2];
            const float gap = pid > -1 ? m.pair_gap[pid] : m.geom_gap[g1] + m.geom_gap[g2];
            CGeom a, b;
            a.pos = ld3(gxpos + 3 * g1); a.rot = gxmat + 9 * g1; a.size = ld3(m.geom_size + 3 * g1); a.margin = margin; a.type = m.geom_type[g1];
            b.pos = ld3(gxpos + 3 * g2); b.rot = gxmat + 9 * g2; b.size = ld3(m.geom_size + 3 * g2); b.margin = margin; b.type = m.geom_type[g2];
#if CCD_MESH
            fill_mesh(m, g1, a); fill_mesh(m, g2, b);
#endif
            bool eovf = false;
            const int nc = ccd_pair(m.ccd_tolerance, gap, m.ccd_iterations, m.epa_iterations, a, b, ccd_scratch + slot * sw, &dist, w1, w2, &eovf);
            if (eovf) ovf |= OVF_EPA_HORIZON;
            if (nc > 0 && dist < gap) {  // collision_convex.py:860-868, 935-943
              dist += margin;
              nrm = dist <= margin ? w1[0] - w2[0] : w2[0] - w1[0];
              if (dist < margin + gap) nhit = nc;  // write_contact
            }
          }
          // pairs keep their list order: exclusive scan of the per-lane contact counts over the batch
          int before = 0, total = 0;
          for (unsigned bb = batch; bb; bb &= bb - 1) {
            const int src = __ffs(bb) - 1;
            const int c = __shfl_sync(FULL_MASK, nhit, src);
            if (src < lane) before += c;
            total += c;
          }
          for (int k = 0; k < nhit; k++) {
            const int off = ncon + before + k;
            if (off < ccap) {
              float* st = stage + STAGE_WORDS * off;
              st[0] = dist; st3(st + 1, (w1[k] + w2[k]) * 0.5f);
              make_frame(nrm, st + 4);
              sgeom[4 * off] = g1; sgeom[4 * off + 1] = g2; sgeom[4 * off + 2] = k; sgeom[4 * off + 3] = pid;
            }
          }
          ncon += total;
          __syncwarp();  // the next batch hands the polytope slots to other lanes
        }
      }
    }
    ovf = __reduce_or_sync(FULL_MASK, (unsigned)ovf);
  }
#pragma unroll 1
  for (int s0 = 0; s0 < nsurv; s0 += 32) {
    const int si = s0 + lane;
    float cd[MAXC];
    v3 cp[MAXC], cn[MAXC];
#pragma unroll
    for (int k = 0; k < MAXC; k++) cd[k] = INFINITY;
    float frame0[9];
    bool shared_frame = false;
    int g1 = 0, g2 = 0;
    float inc = 0.f;  // margin + gap
    int pid = -1;     // explicit pair id of this geom pair, -1 for dynamically generated pairs
    if (si < nsurv) {
      const int e = surv[si];
      g1 = m.nxn_geom_pair[2 * e]; g2 = m.nxn_geom_pair[2 * e + 1];
      if (m.geom_type[g1] > m.geom_type[g2]) { const int t = g1; g1 = g2; g2 = t; }
      const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
      pid = m.npair > 0 ? m.nxn_pairid[2 * e] : -1;
      const float margin = pid > -1 ? m.pair_margin[pid] : m.geom_margin[g1] + m.geom_margin[g2];
      inc = margin + (pid > -1 ? m.pair_gap[pid] : m.geom_gap[g1] + m.geom_gap[g2]);
      const v3 pos1 = ld3(gxpos + 3 * g1), pos2 = ld3(gxpos + 3 * g2);
      const v3 ax1 = matcol(gxmat + 9 * g1, 2), ax2 = matcol(gxmat + 9 * g2, 2);
      const v3 size1 = ld3(m.geom_size + 3 * g1), size2 = ld3(m.geom_size + 3 * g2);
      if (t1 == GEOM_PLANE && t2 == GEOM_SPHERE) {
        cd[0] = plane_sphere(ax1, pos1, pos2, size2.x, &cp[0]); cn[0] = ax1;
      } else if (t1 == GEOM_PLANE && t2 == GEOM_CAPSULE) {
        v3 b = ax2 - ax1 * dot(ax1, ax2);
        const float bn = length(b);
        if (bn != 0.f) b = b * (1.0f / bn);
        if (bn < 0.5f) b = (-0.5f < ax1.y && ax1.y < 0.5f) ? mk3(0.f, 1.f, 0.f) : mk3(0.f, 0.f, 1.f);
        st3(frame0, ax1); st3(frame0 + 3, b); st3(frame0 + 6, cross(ax1, b));
        shared_frame = true;
        const v3 seg = ax2 * size2.y;
        cd[0] = plane_sphere(ax1, pos1, pos2 + seg, size2.x, &cp[0]);
        cd[1] = plane_sphere(ax1, pos1, pos2 - seg, size2.x, &cp[1]);
      } else if (t1 == GEOM_SPHERE && t2 == GEOM_SPHERE) {
        cd[0] = sphere_sphere(pos1, size1.x, pos2, size2.x, &cp[0], &cn[0]);
      } else if (t1 == GEOM_SPHERE && t2 == GEOM_CAPSULE) {
        const v3 seg = ax2 * size2.y;
        const v3 pt = closest_segment_point(pos2 - seg, pos2 + seg, pos1);
        cd[0] = sphere_sphere(pos1, size1.x, pt, size2.x, &cp[0], &cn[0]);
      } else if (t1 == GEOM_CAPSULE && t2 == GEOM_CAPSULE) {
        const v3 axis1 = ax1 * size1.y, axis2 = ax2 * size2.y, dif = pos1 - pos2;
        const float ma = dot(axis1, axis1), mb = -dot(axis1, axis2), mc = dot(axis2, axis2), u = -dot(axis1, dif), v = dot(axis2, dif);
        const float det = ma * mc - mb * mb;
        v3 p, n;
        if (fabsf(det) >= MJ_MINVAL) {
          const float inv = 1.0f / det;
          float x1 = (mc * u - mb * v) * inv, x2 = (ma * v - mb * u) * inv;
          if (x1 > 1.f) { x1 = 1.f; x2 = (v - mb) / mc; } else if (x1 < -1.f) { x1 = -1.f; x2 = (v + mb) / mc; }
          if (x2 > 1.f) { x2 = 1.f; x1 = clampf((u - mb) / ma, -1.f, 1.f); } else if (x2 < -1.f) { x2 = -1.f; x1 = clampf((u + mb) / ma, -1.f, 1.f); }
          const float dist = sphere_sphere(pos1 + axis1 * x1, size1.x, pos2 + axis2 * x2, size2.x, &p, &n);
          if (dist <= margin) { cd[0] = dist; cp[0] = p; cn[0] = n; }
        } else {
          int cc = 0;
          float dist = sphere_sphere(pos1 + axis1, size1.x, pos2 + axis2 * clampf((v - mb) / mc, -1.f, 1.f), size2.x, &p, &n);
          if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; cc++; }
          dist = sphere_sphere(pos1 - axis1, size1.x, pos2 + axis2 * clampf((v + mb) / mc, -1.f, 1.f), size2.x, &p, &n);
          if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; cc++; }
          if (cc < 2) {
            dist = sphere_sphere(pos1 + axis1 * clampf((u - mb) / ma, -1.f, 1.f), size1.x, pos2 + axis2, size2.x, &p, &n);
            if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; cc++; }
          }
          if (cc < 2) {
            dist = sphere_sphere(pos1 + axis1 * clampf((u + mb) / ma, -1.f, 1.f), size1.x, pos2 - axis2, size2.x, &p, &n);
            if (dist <= margin) { cd[cc] = dist; cp[cc] = p; cn[cc] = n; }
          }
        }
      } else if (MAXC >= 8) {
        const float *rot1 = gxmat + 9 * g1, *rot2 = gxmat + 9 * g2;
        if (t1 == GEOM_PLANE && t2 == GEOM_ELLIPSOID) {
          cd[0] = plane_ellipsoid(ax1, pos1, pos2, rot2, size2, &cp[0]); cn[0] = ax1;
        } else if (t1 == GEOM_PLANE && t2 == GEOM_CYLINDER) {
          plane_cylinder(ax1, pos1, pos2, ax2, size2.x, size2.y, cd, cp);
          for (int k = 0; k < 4; k++) cn[k] = ax1;
        } else if (t1 == GEOM_PLANE && t2 == GEOM_BOX) {
          plane_box(ax1, pos1, pos2, rot2, size2, cd, cp);
          for (int k = 0; k < MAXC; k++) cn[k] = ax1;
#if CCD_MESH
        } else if (t1 == GEOM_PLANE && t2 == GEOM_MESH) {  // collision_primitive.py:838 plane_convex: up to four hull vertices below the plane
          CGeom c;
          c.pos = pos2; c.rot = rot2; c.size = size2; c.margin = 0.f; c.type = GEOM_MESH;
          fill_mesh(m, g2, c);
          float d4[4]; v3 p4[4];
          plane_mesh(ax1, pos1, c, d4, p4);
          for (int k = 0; k < 4; k++) { cd[k] = d4[k] < MJ_MAXVAL ? d4[k] : INFINITY; cp[k] = p4[k]; cn[k] = ax1; }
#endif
        } else if (t1 == GEOM_SPHERE && t2 == GEOM_CYLINDER) {
          cd[0] = sphere_cylinder(pos1, size1.x, pos2, ax2, size2.x, size2.y, &cp[0], &cn[0]);
        } else if (t1 == GEOM_SPHERE && t2 == GEOM_BOX) {
          cd[0] = sphere_box(pos1, size1.x, pos2, rot2, size2, &cp[0], &cn[0]);
        } else if (t1 == GEOM_CAPSULE && t2 == GEOM_BOX) {
          capsule_box(pos1, ax1, size1.x, size1.y, pos2, rot2, size2, cd, cp, cn);
        } else if (t1 == GEOM_BOX && t2 == GEOM_BOX && (m.disableflags & DSBL_NATIVECCD)) {  // primitive box-box only with native CCD disabled
          v3 nn;
          const int nc = box_box(pos1, rot1, size1, pos2, rot2, size2, margin, cd, cp, &nn);
          for (int k = 0; k < MAXC; k++) { cn[k] = nn; if (k >= nc) cd[k] = INFINITY; }
        }
      }
    }
    int cnt = 0;  // write_contact: detected = dist < margin + gap
#pragma unroll
    for (int k = 0; k < MAXC; k++) cnt += cd[k] < inc ? 1 : 0;
    int off = ncon + warp_excl_scan(cnt, lane);
    ncon += warp_sum_i(cnt);
#pragma unroll
    for (int k = 0; k < MAXC; k++) {
      if (cd[k] < inc) {
        if (off < ccap) {
          float* st = stage + STAGE_WORDS * off;
          st[0] = cd[k]; st3(st + 1, cp[k]);
          if (shared_frame) { for (int q = 0; q < 9; q++) st[4 + q] = frame0[q]; } else make_frame(cn[k], st + 4);
          sgeom[4 * off] = g1; sgeom[4 * off + 1] = g2; sgeom[4 * off + 2] = k; sgeom[4 * off + 3] = pid;
        }
        off++;
      }
    }
  }
  if (ncon > ccap) { ncon = ccap; ovf |= OVF_NARROWPHASE; }
  __syncwarp();

  // ---- claim one contiguous block of the global pool
  int base = 0;
  if (lane == 0) {
    atomicAdd(d.ncollision, ntotal);
    base = ncon > 0 ? atomicAdd(d.nacon, ncon) : 0;
  }
  base = __shfl_sync(FULL_MASK, base, 0);
  int nwrite = ncon;
  if (base + ncon > d.naconmax) { nwrite = max(0, d.naconmax - base); ovf |= OVF_NARROWPHASE; }
  if (lane == 0) {
    d.world_conadr[w] = base; d.world_ncon[w] = nwrite;
    if (ovf) d.overflow[w] |= ovf;
  }
  const int np = m.nmaxpyramid;
#pragma unroll 1
  for (int c = lane; c < nwrite; c += 32) {
    const int cid = base + c, g1 = sgeom[4 * c], g2 = sgeom[4 * c + 1];
    const float* st = stage + STAGE_WORDS * c;
    ConParams p;
    contact_params(m, g1, g2, sgeom[4 * c + 3], &p);
    d.contact_dist[cid] = st[0];
    for (int k = 0; k < 3; k++) d.contact_pos[3 * cid + k] = st[1 + k];
    for (int k = 0; k < 9; k++) d.contact_frame[9 * cid + k] = st[4 + k];
    d.contact_includemargin[cid] = p.margin;
    for (int k = 0; k < 5; k++) d.contact_friction[5 * cid + k] = p.friction[k];
    d.contact_solref[2 * cid] = p.solref[0]; d.contact_solref[2 * cid + 1] = p.solref[1];
    d.contact_solreffriction[2 * cid] = p.solreffriction[0]; d.contact_solreffriction[2 * cid + 1] = p.solreffriction[1];
    for (int k = 0; k < 5; k++) d.contact_solimp[5 * cid + k] = p.solimp[k];
    d.contact_dim[cid] = p.condim;
    d.contact_geom[2 * cid] = g1; d.contact_geom[2 * cid + 1] = g2;
    for (int k = 0; k < np; k++) d.contact_efc_address[np * cid + k] = -1;
    d.contact_worldid[cid] = w;
    d.contact_type[cid] = CONTACT_TYPE_CONSTRAINT;
    d.contact_geomcollisionid[cid] = sgeom[4 * c + 2];
  }
}

}  // namespace

// warps (= worlds) per block: one-warp blocks cap an SM at 32 resident worlds (CTA limit); MJB_WPB_COL overrides
static int collision_wpb() {
  static int v = 0;
  if (!v) { const char* e = getenv("MJB_WPB_COL"); v = e ? atoi(e) : 2; if (v < 1 || v > 2) v = 2; }
  return v;
}

#ifdef MJB_COLLISION_MESH_TU
#define LAUNCH_NAME launch_collision_mesh
#define SMEM_NAME smem_collision_mesh
#else
#define LAUNCH_NAME launch_collision
#define SMEM_NAME smem_collision
#endif

size_t SMEM_NAME(const ModelDev& m, const DataDev& d) {
#ifndef MJB_COLLISION_MESH_TU
  if (m.nmesh > 0) return smem_collision_mesh(m, d);
#endif
  return (size_t)col_layout(m, d).total * sizeof(float) * collision_wpb();
}

#ifndef MJB_COLLISION_MESH_TU
cudaError_t reset_contact_counters(const DataDev& d, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(d.nacon, 0, sizeof(int), s);
  if (e != cudaSuccess) return e;
  return cudaMemsetAsync(d.ncollision, 0, sizeof(int), s);
}
#endif

cudaError_t LAUNCH_NAME(const ModelDev& m, const DataDev& d, cudaStream_t s) {
#ifndef MJB_COLLISION_MESH_TU
  if (m.nmesh > 0) return launch_collision_mesh(m, d, s);  // models with mesh geoms run the CCD_MESH build of this kernel
#endif
  const size_t smem = SMEM_NAME(m, d);
  static size_t configured4[4] = {0, 0, 0, 0};
#ifdef MJB_COLLISION_MESH_TU
  const int full = 1;
  void (*kern)(ModelDev, DataDev) = m.batched ? k_collision<8, true> : k_collision<8, false>;
#else
  const int full = m.has_multicontact_geom ? 1 : 0;
  void (*kern)(ModelDev, DataDev) = full ? (m.batched ? k_collision<8, true> : k_collision<8, false>) : (m.batched ? k_collision<2, true> : k_collision<2, false>);
#endif
  const int ci = full + 2 * (m.batched ? 1 : 0);
  if (smem > 48 * 1024 && smem > configured4[ci]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured4[ci] = smem;
  }
  const int grid = (d.wn + collision_wpb() - 1) / collision_wpb();
  kern<<<grid, collision_wpb() * 32, smem, s>>>(m, d);
  return cudaGetLastError();
}
