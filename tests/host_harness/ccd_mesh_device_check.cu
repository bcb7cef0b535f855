// Test-only: the CCD_MESH build of mjb_ccd.cuh must compile as device code for sm_90a (tests/test_device_ccd_mesh_on_host.py runs nvcc -c on
// this file).  One thread per pair, geoms given by descriptor -- the shape the collision kernel's convex pass will call it in.
#define CCD_MESH 1
#include "../../mujoco_warp_b200/csrc/mjb_ccd.cuh"

struct DGeomDesc {
  int type, vertnum, polynum, pad;
  const float *size, *pos, *mat, *vert, *polynormal;
  const int *graph, *polyvertadr, *polyvertnum, *polyvert, *polymapadr, *polymapnum, *polymap;
};
__device__ CGeom from_desc(const DGeomDesc& d, float margin) {
  CGeom c;
  c.pos = ld3(d.pos); c.rot = d.mat; c.size = ld3(d.size); c.margin = margin; c.type = d.type;
  c.index = -1; c.vertnum = d.vertnum; c.polynum = d.polynum; c.vert = d.vert; c.polynormal = d.polynormal; c.graph = d.graph;
  c.polyvertadr = d.polyvertadr; c.polyvertnum = d.polyvertnum; c.polyvert = d.polyvert;
  c.polymapadr = d.polymapadr; c.polymapnum = d.polymapnum; c.polymap = d.polymap;
  return c;
}
__global__ void k_ccd_mesh_pairs(const DGeomDesc* g1, const DGeomDesc* g2, int npair, float tolerance, int gjk_it, int epa_it, float* scratch, float* dist,
                                 float* w1, float* w2, int* ncon, int* overflow) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npair) return;
  v3 x1[4], x2[4];
  bool ovf = false;
  float d = 0.f;
  const int n = ccd_pair(tolerance, 1e30f, gjk_it, epa_it, from_desc(g1[p], 0.f), from_desc(g2[p], 0.f), scratch + (size_t)p * ccd_scratch_words(max(gjk_it, epa_it)), &d, x1,
                         x2, &ovf);
  dist[p] = d; ncon[p] = n; overflow[p] = ovf;
  for (int k = 0; k < 4; k++) { st3(w1 + 12 * p + 3 * k, x1[k]); st3(w2 + 12 * p + 3 * k, x2[k]); }
}
