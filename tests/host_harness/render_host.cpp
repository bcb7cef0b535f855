// Test-only: compiles the renderer's per-pixel header (mujoco_warp_b200/csrc/mjb_render.cuh) as plain host C++, so that the device
// source of the camera rays, the geom bounds and the lighting runs on the CPU (tests/test_render_host.py).  Nothing in the product
// path uses this file.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>
using std::max;
using std::min;
static inline float __shfl_xor_sync(unsigned, float v, int) { return v; }
static inline int __shfl_xor_sync(unsigned, int v, int) { return v; }
static inline int __shfl_up_sync(unsigned, int v, int) { return v; }
#include "../../mujoco_warp_b200/csrc/mjb_render.cuh"

// render_compute_ray for n pixels: args (n, 9) = projection, fovy, sensor w, sensor h, img_w, img_h, px, py, znear; intrinsic (n, 4)
extern "C" void hrender_rays(int n, const float* args, const float* intrinsic, float* out) {
  for (int i = 0; i < n; i++) {
    const float* a = args + 9 * i;
    st3(out + 3 * i, render_compute_ray((int)a[0], a[1], a[2], a[3], intrinsic + 4 * i, (int)a[4], (int)a[5], (int)a[6], (int)a[7], a[8]));
  }
}

// render_lighting without shadows for n cases: light (n, 20) = active, type, castshadow, pos[3], dir[3], attenuation[3], cutoff (rad),
// exponent, diffuse[3], specular[3]; surf (n, 11) = normal[3], hit[3], view[3], mat_spec, mat_shin_exp; flags (n, 3) =
// enable_specular, default_attenuation, has_spot; out (n, 6) = diffuse, specular
extern "C" void hrender_lighting(int n, const float* light, const float* surf, const int* flags, float* out) {
  for (int i = 0; i < n; i++) {
    const float* l = light + 20 * i;
    const float* s = surf + 11 * i;
    RenderLight L;
    L.active = l[0] != 0.f; L.type = (int)l[1]; L.castshadow = l[2] != 0.f;
    L.pos = ld3(l + 3); L.dir = ld3(l + 6); L.attenuation = ld3(l + 9); L.cutoff = l[12]; L.exponent = l[13];
    L.diffuse = ld3(l + 14); L.specular = ld3(l + 17);
    v3 df, sp;
    render_lighting(L, ld3(s), ld3(s + 3), ld3(s + 6), s[9], s[10], false, flags[3 * i] != 0, flags[3 * i + 1] != 0, flags[3 * i + 2] != 0, RenderNoShadow(), &df, &sp);
    st3(out + 6 * i, df);
    st3(out + 6 * i + 3, sp);
  }
}

// render_bounds for n geoms: type (n); pos (n, 3), mat (n, 9), size (n, 3), half (n, 3); out (n, 6) = lower, upper
extern "C" void hrender_bounds(int n, const int* type, const float* pos, const float* mat, const float* size, const float* half, float* out) {
  for (int i = 0; i < n; i++) {
    v3 lo, hi;
    render_bounds(type[i], ld3(pos + 3 * i), mat + 9 * i, ld3(size + 3 * i), ld3(half + 3 * i), &lo, &hi);
    st3(out + 6 * i, lo);
    st3(out + 6 * i + 3, hi);
  }
}
