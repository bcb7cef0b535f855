// k_render.cu -- the batch renderer: geom bounds (refit) and one image per (world, active camera).
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): bvh.py:39 refit_bvh and render.py:656 render, without textures, skybox,
// splats, height fields or flex.  The reference traverses a BVH over each world's geom bounds; here every thread tests its pixel's
// ray against all of the world's enabled geoms, culling each by the same bounds first (a BVH only prunes candidates, so the closest
// hit is the same).  One block (blockIdx.x = world, blockIdx.y = tile) takes 128 consecutive pixels of one world (they may span cameras) and stages that world's enabled
// geoms -- type, pose, size, bounds -- in shared memory once; every thread then scans the staged list in ascending order, so ties go
// to the lower geom id and the geom-type branch is uniform across the warp.  Each pixel is written once (coalesced), no atomics.
#include "mjb_launch.cuh"
#include "mjb_ray.cuh"
#include "mjb_render.cuh"
#include "../../include/mjb200.h"

namespace {

constexpr int kRenderBlock = 128;
constexpr int kRefitBlock = 128;

struct SGeom {  // one enabled geom of the block's world, staged in shared memory
  float pos[3], mat[9], size[3], lo[3], hi[3];
  int type, dataid;
};

// BAT: per-world Model fields (geom_size)
template <bool BAT>
__global__ void __launch_bounds__(kRefitBlock) k_refit_bvh(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const __grid_constant__ mjbRender rc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.nworld * rc.ngeom) return;
  const int w = i / rc.ngeom, g = rc.geom_id[i - w * rc.ngeom];
  MJB_WORLD_MODEL(w)
  const int type = m.geom_type[g], did = m.geom_dataid[g];
  const v3 pos = ld3(d.geom_xpos + ((size_t)w * m.ngeom + g) * 3);
  v3 lo = pos, hi = pos;  // bvh.py:217: a mesh geom without mesh data has a point for bounds
  if (type != GEOM_MESH || did >= 0)
    render_bounds(type, pos, d.geom_xmat + ((size_t)w * m.ngeom + g) * 9, ld3(m.geom_size + 3 * g), type == GEOM_MESH ? ld3(rc.mesh_half + 3 * did) : ray_zero3(), &lo, &hi);
  st3(rc.lower + 3 * (size_t)i, lo);
  st3(rc.upper + 3 * (size_t)i, hi);
}

// The ray from pnt against staged geom s in the geom's own routine: distance (-1 on a miss) and world-frame normal
template <bool MESH>
__device__ __forceinline__ float render_geom_at(const ModelDev& m, const SGeom& s, v3 pnt, v3 vec, bool cull, v3* n) {
  const v3 pos = mk3(s.pos[0], s.pos[1], s.pos[2]);
  float x;
  if (MESH && s.type == GEOM_MESH) {
    if (s.dataid < 0) return -1.f;  // no mesh data: nothing to hit
    int f0, f1;
    ray_mesh_range(m, s.dataid, &f0, &f1);
    x = ray_mesh_faces(m.mesh_face, f0, f1, m.mesh_vert + 3 * m.mesh_vertadr[s.dataid], pos, s.mat, pnt, vec, n);
    *n = normalize(*n);
  } else {
    x = ray_geom<true>(pos, s.mat, mk3(s.size[0], s.size[1], s.size[2]), pnt, vec, s.type, n);
  }
  if (cull && x >= 0.f && dot(vec, *n) > 0.f) x = -1.f;
  return x;
}

// The ray against staged geom k: distance (-1 on a miss) and world-frame normal, with render.py:493-497's back-face rule.  The
// quadratics of the sphere, capsule, ellipsoid and cylinder routines lose about (distance / size)^2 ulps to cancellation when solved
// from a far origin, so the ray starts one bounds-width before the point where it enters the geom's bounds (`enter` along it; still
// outside the bounds, so no surface lies between it and the origin), and the distance is that start plus the root.
template <bool MESH>
__device__ __forceinline__ float render_geom(const ModelDev& m, const SGeom& s, v3 pnt, v3 vec, float enter, bool cull, v3* n) {
  const float width = fmaxf(fmaxf(s.hi[0] - s.lo[0], s.hi[1] - s.lo[1]), s.hi[2] - s.lo[2]);
  const float t0 = fmaxf(enter - width, 0.f);
  const float x = render_geom_at<MESH>(m, s, pnt + vec * t0, vec, cull, n);
  return x >= 0.f ? x + t0 : x;
}

// MESH: meshes among the enabled geoms; SHADOW: use_shadows; SPEC / EMIS: enable_specular / enable_emission; BAT: per-world Model fields
template <bool MESH, bool SHADOW, bool SPEC, bool EMIS, bool BAT>
__global__ void __launch_bounds__(kRenderBlock, 4) k_render(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const __grid_constant__ mjbRender rc) {
  extern __shared__ SGeom sg[];
  const int w = blockIdx.x;
  MJB_WORLD_MODEL(w)
  const float* xpos = d.geom_xpos + (size_t)w * m.ngeom * 3;
  const float* xmat = d.geom_xmat + (size_t)w * m.ngeom * 9;
  for (int k = threadIdx.x; k < rc.ngeom; k += blockDim.x) {
    const int g = rc.geom_id[k];
    SGeom& s = sg[k];
    for (int j = 0; j < 3; j++) {
      s.pos[j] = xpos[3 * g + j];
      s.size[j] = m.geom_size[3 * g + j];
      s.lo[j] = rc.lower[((size_t)w * rc.ngeom + k) * 3 + j];
      s.hi[j] = rc.upper[((size_t)w * rc.ngeom + k) * 3 + j];
    }
    for (int j = 0; j < 9; j++) s.mat[j] = xmat[9 * g + j];
    s.type = m.geom_type[g];
    s.dataid = m.geom_dataid[g];
  }
  __syncthreads();

  const int pix = blockIdx.y * blockDim.x + threadIdx.x;
  if (pix >= rc.npixel) return;
  int c = 0;
  while (c + 1 < rc.ncam && pix >= rc.pix_adr[c + 1]) c++;
  const int p = pix - rc.pix_adr[c];
  const int rgb_adr = rc.rgb_adr[c], depth_adr = rc.depth_adr[c], seg_adr = rc.seg_adr[c];
  if (rgb_adr < 0 && depth_adr < 0 && seg_adr < 0) return;
  const int cam = rc.cam_id[c];

  v3 ray_local;
  if (rc.ray) {
    ray_local = ld3(rc.ray + 3 * (size_t)pix);
  } else {
    const int img_w = rc.cam_res[2 * c], img_h = rc.cam_res[2 * c + 1];
    const float* intr = rc.cam_intrinsic + ((size_t)(w % rc.nb_cam_intrinsic) * m.ncam + cam) * 4;
    ray_local = render_compute_ray(rc.cam_projection[cam], rc.cam_fovy[(size_t)(w % rc.nb_cam_fovy) * m.ncam + cam], rc.cam_sensorsize[2 * cam],
                                   rc.cam_sensorsize[2 * cam + 1], intr, img_w, img_h, p % img_w, p / img_w, rc.znear);
  }
  const v3 org = ld3(d.cam_xpos + ((size_t)w * m.ncam + cam) * 3);
  const float* cmat = d.cam_xmat + ((size_t)w * m.ncam + cam) * 9;
  const v3 dir = matvec(cmat, ray_local);
  const v3 inv = mk3(1.0f / dir.x, 1.0f / dir.y, 1.0f / dir.z);
  const bool cull = rc.enable_backface_culling != 0;

  // closest hit (render.py:288 cast_ray)
  float dist = MJ_MAXVAL;
  int hit = -1;
  v3 normal = ray_zero3();
#pragma unroll 1
  for (int k = 0; k < rc.ngeom; k++) {
    const SGeom& s = sg[k];
    float t0;
    if (!render_slab(mk3(s.lo[0], s.lo[1], s.lo[2]), mk3(s.hi[0], s.hi[1], s.hi[2]), org, inv, dist, &t0)) continue;
    v3 n;
    const float x = render_geom<MESH>(m, s, org, dir, t0, cull, &n);
    if (x >= 0.f && x < dist) { dist = x; hit = k; normal = n; }
  }

  const size_t row = (size_t)w;
  if (seg_adr >= 0) {
    int* sp = rc.seg + 2 * (row * rc.nseg + seg_adr + p);
    sp[0] = hit >= 0 ? rc.geom_id[hit] : -1;
    sp[1] = hit >= 0 ? OBJ_GEOM : -1;
  }
  if (depth_adr >= 0) rc.depth[row * rc.ndepth + depth_adr + p] = hit >= 0 ? dist * -ray_local.z : 0.f;
  if (rgb_adr < 0) return;
  if (hit < 0) { rc.rgb[row * rc.nrgb + rgb_adr + p] = rc.background_color; return; }

  // shading (render.py:909-1092)
  const int g = rc.geom_id[hit];
  const v3 hit_point = org + dir * dist;
  const int matid = m.geom_matid[g];
  const float* rgba = matid == -1 ? m.geom_rgba + 4 * g : m.mat_rgba + 4 * matid;
  const v3 base = mk3(rgba[0], rgba[1], rgba[2]);
  float mat_spec = RENDER_DEFAULT_MAT_SPECULAR, mat_shin = 0.5f * RENDER_MAX_SHININESS, mat_emis = RENDER_DEFAULT_MAT_EMISSION;
  if ((SPEC || EMIS) && matid >= 0) {
    if (SPEC) {
      mat_spec = rc.mat_specular[(size_t)(w % rc.nb_mat_specular) * m.nmat + matid];
      mat_shin = rc.mat_shininess[(size_t)(w % rc.nb_mat_shininess) * m.nmat + matid] * RENDER_MAX_SHININESS;
    }
    if (EMIS) mat_emis = rc.mat_emission[(size_t)(w % rc.nb_mat_emission) * m.nmat + matid];
  }
  v3 result = EMIS ? base * mat_emis : ray_zero3();
  const int nl = rc.nlight;
  const float* l_amb = rc.light_ambient + (size_t)(w % rc.nb_light_ambient) * nl * 3;
  if (rc.use_ambient_lighting) {
    if (rc.headlight_active) result = result + mk3(base.x * rc.headlight_ambient[0], base.y * rc.headlight_ambient[1], base.z * rc.headlight_ambient[2]);
    else if (nl == 0) result = result + base * RENDER_NO_LIGHT_AMBIENT;
    if (rc.enable_per_light_ambient)
      for (int l = 0; l < nl; l++)
        if (rc.light_active[l]) result = result + mk3(base.x * l_amb[3 * l], base.y * l_amb[3 * l + 1], base.z * l_amb[3 * l + 2]);
  }
  const v3 view = mk3(-dir.x, -dir.y, -dir.z);
  // any-hit shadow cast (render.py:602-640): every enabled geom the shadow ray enters within max_t
  auto shadow = [&](v3 o, v3 v, float max_t) -> bool {
    if (!SHADOW) return false;
    const v3 iv = mk3(1.0f / v.x, 1.0f / v.y, 1.0f / v.z);
#pragma unroll 1
    for (int k = 0; k < rc.ngeom; k++) {
      const SGeom& s = sg[k];
      float t0;
      if (!render_slab(mk3(s.lo[0], s.lo[1], s.lo[2]), mk3(s.hi[0], s.hi[1], s.hi[2]), o, iv, max_t, &t0)) continue;
      v3 n;
      const float x = render_geom<MESH>(m, s, o, v, t0, cull && !(MESH && s.type == GEOM_MESH), &n);
      if (x >= 0.f && x < max_t) return true;
    }
    return false;
  };
  const float* l_att = rc.light_attenuation + (size_t)(w % rc.nb_light_attenuation) * nl * 3;
  const float* l_cut = rc.light_cutoff + (size_t)(w % rc.nb_light_cutoff) * nl;
  const float* l_exp = rc.light_exponent + (size_t)(w % rc.nb_light_exponent) * nl;
  const float* l_dif = rc.light_diffuse + (size_t)(w % rc.nb_light_diffuse) * nl * 3;
  const float* l_spc = rc.light_specular + (size_t)(w % rc.nb_light_specular) * nl * 3;
#pragma unroll 1
  for (int l = 0; l < nl; l++) {
    RenderLight L;
    L.active = rc.light_active[l] != 0;
    L.castshadow = rc.light_castshadow[l] != 0;
    L.type = rc.light_type[l];
    L.pos = ld3(d.light_xpos + ((size_t)w * nl + l) * 3);
    L.dir = ld3(d.light_xdir + ((size_t)w * nl + l) * 3);
    L.attenuation = ld3(l_att + 3 * l);
    L.cutoff = l_cut[l] * (3.14159265358979f / 180.f);
    L.exponent = l_exp[l];
    L.diffuse = ld3(l_dif + 3 * l);
    L.specular = ld3(l_spc + 3 * l);
    v3 df, sp;
    render_lighting(L, normal, hit_point, view, mat_spec, mat_shin, SHADOW, SPEC, rc.light_attenuation_is_default != 0, rc.has_spot_lights != 0, shadow, &df, &sp);
    result = result + mk3(base.x * df.x, base.y * df.y, base.z * df.z) + sp;
  }
  if (rc.headlight_active) {  // a directional light along the camera's -z that casts no shadow
    RenderLight L;
    L.active = true; L.castshadow = false; L.type = RENDER_LIGHT_DIRECTIONAL;
    L.pos = org;
    L.dir = mk3(-cmat[2], -cmat[5], -cmat[8]);
    L.attenuation = mk3(1.f, 0.f, 0.f);
    L.cutoff = 0.f; L.exponent = 0.f;
    L.diffuse = mk3(rc.headlight_diffuse[0], rc.headlight_diffuse[1], rc.headlight_diffuse[2]);
    L.specular = mk3(rc.headlight_specular[0], rc.headlight_specular[1], rc.headlight_specular[2]);
    v3 df, sp;
    render_lighting(L, normal, hit_point, view, mat_spec, mat_shin, SHADOW, SPEC, true, false, shadow, &df, &sp);
    result = result + mk3(base.x * df.x, base.y * df.y, base.z * df.z) + sp;
  }
  const float r = fmaxf(fminf(result.x, 1.f), 0.f), gg = fmaxf(fminf(result.y, 1.f), 0.f), b = fmaxf(fminf(result.z, 1.f), 0.f);
  rc.rgb[row * rc.nrgb + rgb_adr + p] = render_pack(r * 255.f, gg * 255.f, b * 255.f, 255.f);
}

template <bool MESH, bool SHADOW, bool SPEC, bool EMIS>
void (*render_instance(bool bat))(ModelDev, DataDev, mjbRender) {
  return bat ? k_render<MESH, SHADOW, SPEC, EMIS, true> : k_render<MESH, SHADOW, SPEC, EMIS, false>;
}

template <bool MESH, bool SHADOW>
void (*render_instance(bool spec, bool emis, bool bat))(ModelDev, DataDev, mjbRender) {
  return spec ? (emis ? render_instance<MESH, SHADOW, true, true>(bat) : render_instance<MESH, SHADOW, true, false>(bat))
              : (emis ? render_instance<MESH, SHADOW, false, true>(bat) : render_instance<MESH, SHADOW, false, false>(bat));
}

// render_util.py:255 _build_rays: the camera-frame ray of every pixel of every active camera from the fields' entry 0 (the model's
// values, as the reference takes them from the MjModel)
__global__ void k_render_rays(const __grid_constant__ mjbRender rc, float* __restrict__ ray) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= rc.npixel) return;
  int c = 0;
  while (c + 1 < rc.ncam && pix >= rc.pix_adr[c + 1]) c++;
  const int p = pix - rc.pix_adr[c], cam = rc.cam_id[c], img_w = rc.cam_res[2 * c], img_h = rc.cam_res[2 * c + 1];
  st3(ray + 3 * (size_t)pix, render_compute_ray(rc.cam_projection[cam], rc.cam_fovy[cam], rc.cam_sensorsize[2 * cam], rc.cam_sensorsize[2 * cam + 1],
                                                rc.cam_intrinsic + 4 * cam, img_w, img_h, p % img_w, p / img_w, rc.znear));
}

}  // namespace

cudaError_t launch_render_rays(const mjbRender& rc, float* ray, cudaStream_t s) {
  if (rc.npixel <= 0) return cudaSuccess;
  return launch(k_render_rays, (unsigned)((rc.npixel + kRenderBlock - 1) / kRenderBlock), kRenderBlock, 0, s, rc, ray);
}

size_t smem_render(int ngeom) { return (size_t)ngeom * sizeof(SGeom); }

cudaError_t launch_refit_bvh(const ModelDev& m, const DataDev& d, const mjbRender& rc, cudaStream_t s) {
  const long long n = (long long)d.nworld * rc.ngeom;
  if (n <= 0) return cudaSuccess;
  return launch(m.batched ? k_refit_bvh<true> : k_refit_bvh<false>, (unsigned)((n + kRefitBlock - 1) / kRefitBlock), kRefitBlock, 0, s, m, d, rc);
}

cudaError_t launch_render(const ModelDev& m, const DataDev& d, const mjbRender& rc, bool has_mesh, cudaStream_t s) {
  if (d.nworld <= 0 || rc.npixel <= 0) return cudaSuccess;
  const bool spec = rc.enable_specular != 0, emis = rc.enable_emission != 0, bat = m.batched != 0;
  void (*kern)(ModelDev, DataDev, mjbRender) =
      has_mesh ? (rc.use_shadows ? render_instance<true, true>(spec, emis, bat) : render_instance<true, false>(spec, emis, bat))
               : (rc.use_shadows ? render_instance<false, true>(spec, emis, bat) : render_instance<false, false>(spec, emis, bat));
  const dim3 grid((unsigned)d.nworld, (unsigned)((rc.npixel + kRenderBlock - 1) / kRenderBlock));  // the caller bounds the tiles by 65535
  const cudaError_t e = launch_configure((const void*)kern, smem_render(rc.ngeom));
  if (e != cudaSuccess) return e;
  kern<<<grid, kRenderBlock, smem_render(rc.ngeom), s>>>(m, d, rc);
  g_launches++;
  return cudaGetLastError();
}
