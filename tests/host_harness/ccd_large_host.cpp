// Test-only: compiles mjb_ccd.cuh as plain host C++ with CCD_MESH=2, the mesh build whose multi-contact buffers are scratch sized from the
// model (the build k_collision_mesh_large.cu and k_sensor_collision_large.cu run), so that it can be checked against the oracle and the
// reference fixtures without a GPU.  Same descriptor layout as ccd_host.cpp's hccd_desc.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <algorithm>
#ifndef __noinline__
#define __noinline__
#endif
using std::max;
using std::min;
// warp intrinsics referenced by helpers in mjb_math.cuh that the pair routines never call
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
static inline float __shfl_sync(unsigned, float v, int) { return v; }
static inline int __shfl_sync(unsigned, int v, int) { return v; }
static inline unsigned __ballot_sync(unsigned, int p) { return p ? 1u : 0u; }
static inline void __syncwarp(unsigned = 0xffffffffu) {}
#include "../../mujoco_warp_b200/csrc/mjb_ccd.cuh"

struct HGeomDesc {
  int type, vertnum, polynum, pad;
  const float *size, *pos, *mat, *vert, *polynormal;
  const int *graph, *polyvertadr, *polyvertnum, *polyvert, *polymapadr, *polymapnum, *polymap;
};
static CGeom from_desc(const HGeomDesc* d, float margin) {
  CGeom c;
  memset(&c, 0, sizeof c);
  c.pos = ld3(d->pos); c.rot = d->mat; c.size = ld3(d->size); c.margin = margin; c.type = d->type;
  c.index = -1; c.vertnum = d->vertnum; c.polynum = d->polynum; c.vert = d->vert; c.polynormal = d->polynormal; c.graph = d->graph;
  c.polyvertadr = d->polyvertadr; c.polyvertnum = d->polyvertnum; c.polyvert = d->polyvert;
  c.polymapadr = d->polymapadr; c.polymapnum = d->polymapnum; c.polymap = d->polymap;
  return c;
}
// npolygonmax / nmeshdegmax: the model's, as MeshClipDev carries them; the scratch is sized by mesh_clip_words like mjb_data_finalize's and
// fenced by a canary that must survive the call (*overflow bit 1 if it did not)
extern "C" int hccd_large_desc(const HGeomDesc* d1, const HGeomDesc* d2, float margin, float tolerance, float cutoff, int gjk_iterations, int epa_iterations,
                               int npolygonmax, int nmeshdegmax, float* dist, float* w1, float* w2, int* overflow) {
  const CGeom a = from_desc(d1, margin), b = from_desc(d2, margin);
  const int it = std::max(gjk_iterations, epa_iterations);
  float* scratch = new float[ccd_scratch_words(it) + 64]();
  MeshClipDev c;
  memset(&c, 0, sizeof c);
  c.npolygonmax = npolygonmax; c.nmeshdegmax = nmeshdegmax;
  const int words = mesh_clip_words(c), guard = 64;
  float* clip = new float[words + guard];
  for (int k = 0; k < words + guard; k++) clip[k] = -12345.f;
  const CcdClip mc = {clip, mesh_clip_poly(c), mesh_clip_deg(c)};
  v3 x1[4], x2[4];
  memset(x1, 0, sizeof x1); memset(x2, 0, sizeof x2);
  bool ovf = false;
  const int n = ccd_pair(tolerance, cutoff, gjk_iterations, epa_iterations, a, b, scratch, dist, x1, x2, &ovf, mc);
  for (int k = 0; k < 4; k++) { st3(w1 + 3 * k, x1[k]); st3(w2 + 3 * k, x2[k]); }
  *overflow = ovf ? 1 : 0;
  for (int k = words; k < words + guard; k++) if (clip[k] != -12345.f) *overflow |= 2;
  delete[] scratch;
  delete[] clip;
  return n;
}
extern "C" void hplane_mesh_large(const float* n_world, const float* plane_pos, const HGeomDesc* d, float* dist, float* pos) {
  const CGeom c = from_desc(d, 0.f);
  v3 p4[4];
  plane_mesh(ld3(n_world), ld3(plane_pos), c, dist, p4);
  for (int k = 0; k < 4; k++) st3(pos + 3 * k, p4[k]);
}
