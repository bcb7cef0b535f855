// Test-only: compiles the fluid-force header (mujoco_warp_b200/csrc/mjb_fluid.cuh) as plain host C++, so that the device source of the
// inertia-box and ellipsoid models and of the projection to dofs runs on the CPU against the reference-generated fixtures
// (tests/golden/fluid_*.npz).  Nothing in the product path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>
#include <algorithm>
using std::max;
using std::min;
// warp intrinsics mjb_math.cuh's helpers name (unused by the fluid routines)
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
#include "../../mujoco_warp_b200/csrc/mjb_fluid.cuh"

// k_velocity's fluid pass for every world: the body wrenches, then qfrc_fluid (nworld, nv)
extern "C" void hfluid_qfrc(int nv, int nbody, int ngeom, const int* body_rootid, const int* dof_bodyid, const int* body_isdofancestor,
                            const float* body_mass, const float* body_inertia, const int* geom_type, const float* geom_size, const int* body_fluid,
                            const int* body_geomadr, const int* body_geomnum, const float* geom_fluid, float density, float viscosity, const float* wind,
                            int nworld, const float* cvel, const float* xipos, const float* ximat, const float* geom_xpos, const float* geom_xmat,
                            const float* subtree_com, const float* cdof, float* qfrc) {
  ModelDev m;
  memset(&m, 0, sizeof m);
  m.nv = nv; m.nbody = nbody; m.ngeom = ngeom;
  m.body_rootid = body_rootid; m.dof_bodyid = dof_bodyid; m.body_isdofancestor = body_isdofancestor; m.body_mass = body_mass;
  m.body_inertia = body_inertia; m.geom_type = geom_type; m.geom_size = geom_size;
  FluidDev f;
  memset(&f, 0, sizeof f);
  f.has_fluid = 1; f.density = density; f.viscosity = viscosity; f.wind_x = wind[0]; f.wind_y = wind[1]; f.wind_z = wind[2];
  f.body_fluid = body_fluid; f.body_geomadr = body_geomadr; f.body_geomnum = body_geomnum; f.geom_fluid = geom_fluid;
  float* ft = new float[6 * nbody];
  for (int w = 0; w < nworld; w++) {
    const float *xip = xipos + (size_t)w * nbody * 3, *stc = subtree_com + (size_t)w * nbody * 3;
    for (int b = 0; b < nbody; b++)
      fluid_body_wrench(m, f, b, cvel + ((size_t)w * nbody + b) * 6, ld3(xip + 3 * b), ximat + ((size_t)w * nbody + b) * 9, ld3(stc + 3 * body_rootid[b]),
                        geom_xpos + (size_t)w * ngeom * 3, geom_xmat + (size_t)w * ngeom * 9, ft + 6 * b);
    for (int dd = 0; dd < nv; dd++) qfrc[(size_t)w * nv + dd] = fluid_project(m, dd, cdof + ((size_t)w * nv + dd) * 6, ft, xip, stc);
  }
  delete[] ft;
}
