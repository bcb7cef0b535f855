// mjb_render.cuh -- per-pixel arithmetic of the batch renderer (k_render.cu): camera rays, geom bounds and Phong lighting (fp32).
//
// Restates the reference's render_util.py:71 compute_ray and :133 pack_rgba_to_uint32, bvh.py:47-174 (the bounds of each geom type)
// and render.py:518 compute_lighting, in their operation order.  Scalar code, one pixel per thread: compiles as plain host C++ too
// (tests/host_harness/render_host.cpp).
#pragma once
#include "mjb_math.cuh"
#include "mjb_types.cuh"

#define RENDER_MAX_SHININESS 128.0f             // render.py:159: 8-bit output, so the Phong exponent tops out at 128
#define RENDER_DEFAULT_MAT_SPECULAR 0.5f        // :164, MuJoCo's default mat_specular
#define RENDER_DEFAULT_MAT_EMISSION 0.0f        // :167
#define RENDER_NO_LIGHT_AMBIENT 0.3f            // :169: ambient of a model without lights, and the light left in a shadow
#define RENDER_PLANE_EXTENT 1000.0f             // bvh.py:112: half-extent of an infinite plane's bounds
enum { RENDER_LIGHT_SPOT = 0, RENDER_LIGHT_DIRECTIONAL = 1 };

// render_util.py:71 compute_ray: unit direction of pixel (px, py) of an img_w x img_h image, in the camera frame (looking along -z)
static __device__ __forceinline__ v3 render_compute_ray(int projection, float fovy, float sensor_w, float sensor_h, const float* intrinsic, int img_w, int img_h,
                                                        int px, int py, float znear) {
  if (projection == 1) return mk3(0.f, 0.f, -1.f);  // orthographic
  const float aspect = (float)img_w / (float)img_h;
  float left, right, top, bottom;
  if (sensor_h != 0.f) {
    const float fx = intrinsic[0], fy = intrinsic[1], cx = intrinsic[2], cy = intrinsic[3];
    const float sensor_aspect = sensor_w / sensor_h;
    if (aspect > sensor_aspect) sensor_h = sensor_w / aspect;
    else if (aspect < sensor_aspect) sensor_w = sensor_h * aspect;
    const float ifx = znear / fx, ify = znear / fy;
    left = -ifx * (sensor_w * 0.5f - cx);
    right = ifx * (sensor_w * 0.5f + cx);
    top = ify * (sensor_h * 0.5f - cy);
    bottom = -ify * (sensor_h * 0.5f + cy);
  } else {
    const float half_h = znear * tanf(0.5f * (fovy * (3.14159265358979f / 180.f)));
    const float half_w = half_h * aspect;
    left = -half_w; right = half_w; top = half_h; bottom = -half_h;
  }
  const float u = ((float)px + 0.5f) / (float)img_w, v = ((float)py + 0.5f) / (float)img_h;
  return normalize(mk3(left + (right - left) * u, top + (bottom - top) * v, -znear));
}

// render_util.py:133 pack_rgba_to_uint32 of channels already scaled to [0, 255] (truncated, as int() does)
static __device__ __forceinline__ unsigned render_pack(float r, float g, float b, float a) {
  return ((unsigned)(int)a << 24) | ((unsigned)(int)r << 16) | ((unsigned)(int)g << 8) | (unsigned)(int)b;
}

// bvh.py:178 _compute_bvh_bounds for one geom: `half` is the mesh's vertex-box half-extent (meshes only)
static __device__ __forceinline__ void render_bounds(int type, v3 pos, const float* mat, v3 size, v3 half, v3* lo, v3* hi) {
  float e[3];
  if (type == GEOM_SPHERE) {
    e[0] = e[1] = e[2] = size.x;
  } else if (type == GEOM_CAPSULE) {
    for (int i = 0; i < 3; i++) e[i] = fabsf(mat[3 * i + 2] * size.y) + size.x;
  } else if (type == GEOM_ELLIPSOID) {
    for (int i = 0; i < 3; i++) {
      const float a = mat[3 * i] * size.x, b = mat[3 * i + 1] * size.y, c = mat[3 * i + 2] * size.z;
      e[i] = sqrtf(a * a + b * b + c * c);
    }
  } else if (type == GEOM_CYLINDER) {
    for (int i = 0; i < 3; i++) e[i] = size.x * sqrtf(mat[3 * i] * mat[3 * i] + mat[3 * i + 1] * mat[3 * i + 1]) + size.y * fabsf(mat[3 * i + 2]);
  } else if (type == GEOM_PLANE) {
    // :103 the four corners of a square of half-side 2 max(size x, y) (1000 when infinite), widened by 0.01
    const float sc = (size.x <= 0.f || size.y <= 0.f) ? RENDER_PLANE_EXTENT : fmaxf(size.x, size.y) * 2.0f;
    for (int i = 0; i < 3; i++) e[i] = sc * (fabsf(mat[3 * i]) + fabsf(mat[3 * i + 1])) + 0.01f;
  } else {  // box; mesh with the vertex box's half-extent
    const v3 s = type == GEOM_MESH ? half : size;
    for (int i = 0; i < 3; i++) e[i] = fabsf(mat[3 * i]) * s.x + fabsf(mat[3 * i + 1]) * s.y + fabsf(mat[3 * i + 2]) * s.z;
  }
  *lo = mk3(pos.x - e[0], pos.y - e[1], pos.z - e[2]);
  *hi = mk3(pos.x + e[0], pos.y + e[1], pos.z + e[2]);
}

// Slab test: the ray enters the box [lo, hi] at a distance below max_t (and not only behind its origin); *enter: where it enters, >= 0
static __device__ __forceinline__ bool render_slab(v3 lo, v3 hi, v3 pnt, v3 inv, float max_t, float* enter) {
  const float ax = (lo.x - pnt.x) * inv.x, bx = (hi.x - pnt.x) * inv.x;
  const float ay = (lo.y - pnt.y) * inv.y, by = (hi.y - pnt.y) * inv.y;
  const float az = (lo.z - pnt.z) * inv.z, bz = (hi.z - pnt.z) * inv.z;
  const float tmin = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz));
  const float tmax = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fmaxf(az, bz));
  *enter = fmaxf(tmin, 0.f);
  return tmax >= *enter && tmin < max_t;
}

// One light as render.py:518 compute_lighting takes it (cutoff in radians)
struct RenderLight {
  bool active, castshadow;
  int type;
  v3 pos, dir, attenuation, diffuse, specular;
  float cutoff, exponent;
};

// render.py:518 compute_lighting: the light's diffuse and specular contributions at a surface point.  `shadow(origin, dir, max_t)`
// is the any-hit cast (true: occluded); it is called only with use_shadows and a shadow-casting light.
template <class Shadow>
static __device__ __forceinline__ void render_lighting(const RenderLight& l, v3 normal, v3 hit, v3 view, float mat_spec, float mat_shin_exp, bool use_shadows,
                                                       bool enable_specular, bool default_attenuation, bool has_spot, const Shadow& shadow, v3* diff, v3* spec) {
  *diff = mk3(0.f, 0.f, 0.f);
  *spec = mk3(0.f, 0.f, 0.f);
  if (!l.active) return;
  v3 L;
  float dist_to_light = MJ_MAXVAL, attenuation = 1.0f;
  if (l.type == RENDER_LIGHT_DIRECTIONAL) {
    L = mk3(-l.dir.x, -l.dir.y, -l.dir.z);
  } else {
    const v3 dl = l.pos - hit;
    const float n = length(dl);
    L = dl;
    dist_to_light = 0.f;
    if (n != 0.f) { L = dl * (1.0f / n); dist_to_light = n; }
    if (!default_attenuation) {
      const float den = l.attenuation.x + dist_to_light * l.attenuation.y + dist_to_light * dist_to_light * l.attenuation.z;
      attenuation = 1.0f / (den != 0.f ? den : MJ_MINVAL);
    }
    if (has_spot && l.type == RENDER_LIGHT_SPOT) {
      const float cos_theta = -dot(L, l.dir);
      if (cos_theta < cosf(l.cutoff)) return;
      attenuation = attenuation * powf(fmaxf(cos_theta, 0.f), l.exponent);
    }
  }
  const float ndotl = fmaxf(0.f, dot(normal, L));
  if (ndotl == 0.f) return;
  float visible = 1.0f;
  if (use_shadows && l.castshadow) {
    const float max_t = l.type == RENDER_LIGHT_DIRECTIONAL ? 1.0e8f : dist_to_light - 1.0e-3f;
    if (shadow(hit + normal * 1.0e-4f, L, max_t)) visible = RENDER_NO_LIGHT_AMBIENT;
  }
  const float weight = attenuation * visible;
  *diff = l.diffuse * (ndotl * weight);
  if (enable_specular && mat_spec > 0.f && mat_shin_exp > 0.f) {
    const v3 H = normalize(L + view);
    const float ndoth = fmaxf(0.f, dot(normal, H));
    *spec = l.specular * (mat_spec * powf(ndoth, mat_shin_exp) * weight);
  }
}

// No shadow rays (use_shadows off, and the host build)
struct RenderNoShadow {
  __device__ bool operator()(v3, v3, float) const { return false; }
};
