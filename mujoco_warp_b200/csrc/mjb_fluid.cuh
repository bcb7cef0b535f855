// mjb_fluid.cuh -- forces of a surrounding fluid (density, viscosity, wind) on the bodies, and their velocity derivatives.
//
// Restates the reference (/root/reference/mujoco_warp/_src/) in its operation order: passive.py:46 geom_semiaxes, :63
// ellipsoid_max_moment, :307-528 _fluid_force (the inertia-box model and the ellipsoid model), support.py:259 _apply_ft (the
// projection to dofs), derivative.py:588-868 _deriv_ellipsoid_fluid and :870-933 _deriv_box_fluid (the 6x6 derivative B of the
// local wrench with respect to the local velocity, symmetrized for implicitfast) and :935-966, 1039-1041 (J_i^T B J_j).
// The model's fluid fields come in a FluidDev (mjb_types.cuh).  k_velocity computes the forces (one team lane per body);
// tree_implicit_a (mjb_implicit_a.cuh) adds -dt J_i^T B J_j to A.
//
// Scalar code: compiles as plain host C++ too (tests/host_harness/fluid_host.cpp).
#pragma once
#include "mjb_math.cuh"
#include "mjb_types.cuh"

enum { FLUID_NONE = 0, FLUID_ELLIPSOID = 1, FLUID_BOX = 2 };  // FluidDev.body_fluid

// row-major 3x3 times a vector, and its transpose times a vector
static __device__ __forceinline__ v3 fl_mv(const float* R, v3 v) {
  return mk3(R[0] * v.x + R[1] * v.y + R[2] * v.z, R[3] * v.x + R[4] * v.y + R[5] * v.z, R[6] * v.x + R[7] * v.y + R[8] * v.z);
}
static __device__ __forceinline__ v3 fl_mtv(const float* R, v3 v) {
  return mk3(R[0] * v.x + R[3] * v.y + R[6] * v.z, R[1] * v.x + R[4] * v.y + R[7] * v.z, R[2] * v.x + R[5] * v.y + R[8] * v.z);
}
static __device__ __forceinline__ float fl_comp(v3 v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : v.z); }
static __device__ __forceinline__ float fl_pow2(float v) { return v * v; }
static __device__ __forceinline__ float fl_pow4(float v) { const float s = v * v; return s * s; }

// passive.py:46
static __device__ __forceinline__ v3 fluid_semiaxes(int type, const float* size) {
  if (type == GEOM_SPHERE) return mk3(size[0], size[0], size[0]);
  if (type == GEOM_CAPSULE) return mk3(size[0], size[0], size[1] + size[0]);
  if (type == GEOM_CYLINDER) return mk3(size[0], size[0], size[1]);
  return ld3(size);
}
// passive.py:63
static __device__ __forceinline__ float fluid_max_moment(v3 s, int dir) {
  const float d0 = fl_comp(s, dir), d1 = fl_comp(s, (dir + 1) % 3), d2 = fl_comp(s, (dir + 2) % 3);
  return (float)(8.0 / 15.0 * 3.14159265358979323846) * d0 * fl_pow4(fmaxf(d1, d2));
}

// The body's velocity at its inertial frame origin: angular and linear, world frame (cvel is about the subtree root's com).
static __device__ __forceinline__ void fluid_body_vel(const float* cvel, v3 xipos, v3 root_com, v3* ang, v3* lin) {
  *ang = ld3(cvel);
  *lin = ld3(cvel + 3) - cross(xipos - root_com, *ang);
}

// passive.py:307-528: the world-frame force (ft[0..2]) and torque (ft[3..5]) of the fluid on body b (b > 0).  geom_xpos / geom_xmat
// are the world's arrays, cvel the body's 6 entries.
static __device__ void fluid_body_wrench(const ModelDev& m, const FluidDev& f, int b, const float* cvel, v3 xipos, const float* ximat, v3 root_com,
                                         const float* geom_xpos, const float* geom_xmat, float* ft) {
  const float PI = 3.14159265358979323846f;
  for (int k = 0; k < 6; k++) ft[k] = 0.f;
  const float mass = m.body_mass[b];
  if (b == 0 || mass < MJ_MINVAL || f.body_fluid[b] == FLUID_NONE) return;
  const v3 wind = mk3(f.wind_x, f.wind_y, f.wind_z);
  const bool has_wind = f.wind_x != 0.f || f.wind_y != 0.f || f.wind_z != 0.f;
  const float density = f.density, viscosity = f.viscosity;
  v3 ang_global, lin_com;
  fluid_body_vel(cvel, xipos, root_com, &ang_global, &lin_com);

  if (f.body_fluid[b] == FLUID_ELLIPSOID) {
    v3 force_global = mk3(0.f, 0.f, 0.f), torque_global = mk3(0.f, 0.f, 0.f);
    const int start = f.body_geomadr[b], count = f.body_geomnum[b];
    for (int i = 0; i < count; i++) {
      const int g = start + i;
      const float* fl = f.geom_fluid + 12 * g;
      const float coef = fl[0];
      if (coef <= 0.f) continue;
      const v3 s = fluid_semiaxes(m.geom_type[g], m.geom_size + 3 * g);
      const float* grot = geom_xmat + 9 * g;
      const v3 gpos = ld3(geom_xpos + 3 * g);
      const v3 lin_point = lin_com + cross(ang_global, gpos - xipos);
      const v3 l_ang = fl_mtv(grot, ang_global);
      v3 l_lin = fl_mtv(grot, lin_point);
      if (has_wind) l_lin = l_lin - fl_mtv(grot, wind);
      v3 lfrc_torque = mk3(0.f, 0.f, 0.f), lfrc_force = mk3(0.f, 0.f, 0.f);
      if (density > 0.f) {  // added mass
        const v3 vlm = mk3(density * fl[6] * l_lin.x, density * fl[7] * l_lin.y, density * fl[8] * l_lin.z);
        const v3 vam = mk3(density * fl[9] * l_ang.x, density * fl[10] * l_ang.y, density * fl[11] * l_ang.z);
        lfrc_force = lfrc_force + cross(vlm, l_ang);
        lfrc_torque = lfrc_torque + (cross(vlm, l_lin) + cross(vam, l_ang));
      }
      const float magnus_coef = fl[5], kutta_coef = fl[4], blunt_drag_coef = fl[1], slender_drag_coef = fl[2], ang_drag_coef = fl[3];
      const float volume = (float)(4.0 / 3.0 * 3.14159265358979323846) * s.x * s.y * s.z;
      const float d_max = fmaxf(fmaxf(s.x, s.y), s.z), d_min = fminf(fminf(s.x, s.y), s.z);
      const float d_mid = s.x + s.y + s.z - d_max - d_min;
      const float A_max = PI * d_max * d_mid;
      const float lin_speed = length(l_lin);
      const v3 magnus_force = cross(l_ang, l_lin) * (magnus_coef * density * volume);
      const float s12 = s.y * s.z, s20 = s.z * s.x, s01 = s.x * s.y;
      const float proj_denom = fl_pow4(s12) * fl_pow2(l_lin.x) + fl_pow4(s20) * fl_pow2(l_lin.y) + fl_pow4(s01) * fl_pow2(l_lin.z);
      const float proj_num = fl_pow2(s12 * l_lin.x) + fl_pow2(s20 * l_lin.y) + fl_pow2(s01 * l_lin.z);
      const float A_proj = PI * sqrtf(proj_denom / fmaxf(MJ_MINVAL, proj_num));
      const float cos_alpha = proj_num / fmaxf(MJ_MINVAL, lin_speed * proj_denom);
      const v3 norm = mk3(fl_pow2(s12) * l_lin.x, fl_pow2(s20) * l_lin.y, fl_pow2(s01) * l_lin.z);
      v3 kutta_force = mk3(0.f, 0.f, 0.f);
      if (density > 0.f && kutta_coef != 0.f && lin_speed > MJ_MINVAL) {
        const v3 kutta_circ = cross(norm, l_lin) * (kutta_coef * density * cos_alpha * A_proj);
        kutta_force = cross(kutta_circ, l_lin);
      }
      const float eq_sphere_D = (float)(2.0 / 3.0) * (s.x + s.y + s.z);
      const float lin_visc_force_coef = (float)(3.0 * 3.14159265358979323846) * eq_sphere_D;
      const float lin_visc_torq_coef = PI * eq_sphere_D * eq_sphere_D * eq_sphere_D;
      const float I_max = (float)(8.0 / 15.0 * 3.14159265358979323846) * d_mid * fl_pow4(d_max);
      const float II0 = fluid_max_moment(s, 0), II1 = fluid_max_moment(s, 1), II2 = fluid_max_moment(s, 2);
      const v3 mom_visc = mk3(l_ang.x * (ang_drag_coef * II0 + slender_drag_coef * (I_max - II0)),
                              l_ang.y * (ang_drag_coef * II1 + slender_drag_coef * (I_max - II1)),
                              l_ang.z * (ang_drag_coef * II2 + slender_drag_coef * (I_max - II2)));
      const float drag_lin_coef = viscosity * lin_visc_force_coef + density * lin_speed * (A_proj * blunt_drag_coef + slender_drag_coef * (A_max - A_proj));
      const float drag_ang_coef = viscosity * lin_visc_torq_coef + density * length(mom_visc);
      lfrc_torque = lfrc_torque - drag_ang_coef * l_ang;
      lfrc_force = lfrc_force + (magnus_force + kutta_force - drag_lin_coef * l_lin);
      lfrc_torque = lfrc_torque * coef;
      lfrc_force = lfrc_force * coef;
      torque_global = torque_global + fl_mv(grot, lfrc_torque);
      force_global = force_global + fl_mv(grot, lfrc_force);
    }
    st3(ft, force_global); st3(ft + 3, torque_global);
    return;
  }

  // inertia box
  const v3 l_ang = fl_mtv(ximat, ang_global);
  v3 l_lin = fl_mtv(ximat, lin_com);
  if (has_wind) l_lin = l_lin - fl_mtv(ximat, wind);
  v3 lfrc_torque = mk3(0.f, 0.f, 0.f), lfrc_force = mk3(0.f, 0.f, 0.f);
  const bool has_viscosity = viscosity > 0.f, has_density = density > 0.f;
  float box0 = 0.f, box1 = 0.f, box2 = 0.f;
  if (has_viscosity || has_density) {
    const v3 inertia = ld3(m.body_inertia + 3 * b);
    const float scl = 6.0f / mass;
    box0 = sqrtf(fmaxf(MJ_MINVAL, inertia.y + inertia.z - inertia.x) * scl);
    box1 = sqrtf(fmaxf(MJ_MINVAL, inertia.x + inertia.z - inertia.y) * scl);
    box2 = sqrtf(fmaxf(MJ_MINVAL, inertia.x + inertia.y - inertia.z) * scl);
  }
  if (has_viscosity) {
    const float diam = (box0 + box1 + box2) / 3.0f;
    lfrc_torque = -1.0f * l_ang * powf(diam, 3.0f) * PI * viscosity;
    lfrc_force = -3.0f * l_lin * diam * PI * viscosity;
  }
  if (has_density) {
    lfrc_force = lfrc_force - mk3(0.5f * density * box1 * box2 * fabsf(l_lin.x) * l_lin.x, 0.5f * density * box0 * box2 * fabsf(l_lin.y) * l_lin.y,
                                  0.5f * density * box0 * box1 * fabsf(l_lin.z) * l_lin.z);
    const float scl = density / 64.0f;
    const float b0p4 = powf(box0, 4.0f), b1p4 = powf(box1, 4.0f), b2p4 = powf(box2, 4.0f);
    lfrc_torque = lfrc_torque - mk3(box0 * (b1p4 + b2p4) * fabsf(l_ang.x) * l_ang.x * scl, box1 * (b0p4 + b2p4) * fabsf(l_ang.y) * l_ang.y * scl,
                                    box2 * (b0p4 + b1p4) * fabsf(l_ang.z) * l_ang.z * scl);
  }
  st3(ft, fl_mv(ximat, lfrc_force)); st3(ft + 3, fl_mv(ximat, lfrc_torque));
}

// support.py:259-300 _apply_ft for one dof: the body wrenches ft (6 per body: force, torque) projected on dof dd at each body's
// inertial frame origin, summed over the bodies of the dof's subtree in body order.  cdof: the dof's 6 entries; xipos / subtree_com:
// the world's arrays.
static __device__ __forceinline__ float fluid_project(const ModelDev& m, int dd, const float* cdof, const float* ft, const float* xipos, const float* subtree_com) {
  const int nv = m.nv, nb = m.nbody;
  const v3 cang = ld3(cdof);
  float acc = 0.f;
  for (int b = m.dof_bodyid[dd]; b < nb; b++) {
    const float* w = ft + 6 * b;
    if (w[0] == 0.f && w[1] == 0.f && w[2] == 0.f && w[3] == 0.f && w[4] == 0.f && w[5] == 0.f) continue;
    if (!m.body_isdofancestor[b * nv + dd]) continue;
    const v3 off = ld3(xipos + 3 * b) - ld3(subtree_com + 3 * m.body_rootid[b]);
    const v3 cr = cross(cang, off);
    acc += cdof[3] * w[0] + cdof[4] * w[1] + cdof[5] * w[2] + cdof[0] * w[3] + cdof[1] * w[4] + cdof[2] * w[5] + dot(cr, ld3(w));
  }
  return acc;
}

// derivative.py:870-933 _deriv_box_fluid: B is diagonal (angular 0..2, linear 3..5); symmetrizing leaves it unchanged.
static __device__ __forceinline__ void fluid_box_B(const ModelDev& m, const FluidDev& f, int b, const float* lvel, float* Bd) {
  const float PI = 3.14159265358979323846f;
  const float density = f.density, viscosity = f.viscosity;
  for (int k = 0; k < 6; k++) Bd[k] = 0.f;
  const float mass = m.body_mass[b];
  const v3 inertia = ld3(m.body_inertia + 3 * b);
  const float scl = 6.0f / mass;
  const float box0 = sqrtf(fmaxf(MJ_MINVAL, inertia.y + inertia.z - inertia.x) * scl);
  const float box1 = sqrtf(fmaxf(MJ_MINVAL, inertia.x + inertia.z - inertia.y) * scl);
  const float box2 = sqrtf(fmaxf(MJ_MINVAL, inertia.x + inertia.y - inertia.z) * scl);
  if (viscosity > 0.f) {
    const float diam = (box0 + box1 + box2) * (float)(1.0 / 3.0);
    const float visc_rot = -PI * diam * diam * diam * viscosity, visc_lin = (float)(-3.0 * 3.14159265358979323846) * diam * viscosity;
    Bd[0] += visc_rot; Bd[1] += visc_rot; Bd[2] += visc_rot;
    Bd[3] += visc_lin; Bd[4] += visc_lin; Bd[5] += visc_lin;
  }
  if (density > 0.f) {
    const float t0 = box1 * box1 * box1 * box1 + box2 * box2 * box2 * box2, t1 = box0 * box0 * box0 * box0 + box2 * box2 * box2 * box2,
                t2 = box0 * box0 * box0 * box0 + box1 * box1 * box1 * box1;
    const float inv_32 = (float)(1.0 / 32.0);
    Bd[0] -= density * box0 * t0 * fabsf(lvel[0]) * inv_32;
    Bd[1] -= density * box1 * t1 * fabsf(lvel[1]) * inv_32;
    Bd[2] -= density * box2 * t2 * fabsf(lvel[2]) * inv_32;
    Bd[3] -= density * box1 * box2 * fabsf(lvel[3]);
    Bd[4] -= density * box0 * box2 * fabsf(lvel[4]);
    Bd[5] -= density * box0 * box1 * fabsf(lvel[5]);
  }
}

// derivative.py:588-852 _deriv_ellipsoid_fluid for one geom: B (6 x 6, row-major, rows and columns [angular; linear]) at the geom's
// local velocity, symmetrized as for implicitfast (SYM); without SYM as it stands, as derivative.py:800 leaves it for the other integrators.
template <bool SYM = true>
static __device__ void fluid_ellipsoid_B(const float* fl, v3 s, v3 ang_vel, v3 lin_vel, float density, float viscosity, float* B) {
  const float PI = 3.14159265358979323846f;
  float B00[9], B01[9], B10[9], B11[9];
  for (int k = 0; k < 9; k++) B00[k] = B01[k] = B10[k] = B11[k] = 0.f;
  // skew(v)[r][c]
  auto sk = [](v3 v, int r, int c) -> float {
    const int k = 3 * r + c;
    return k == 1 ? -v.z : k == 2 ? v.y : k == 3 ? v.z : k == 5 ? -v.x : k == 6 ? -v.y : k == 7 ? v.x : 0.f;
  };
  if (density > 0.f) {
    const v3 dvm = mk3(density * fl[6], density * fl[7], density * fl[8]), dvi = mk3(density * fl[9], density * fl[10], density * fl[11]);
    const v3 vlm = mk3(dvm.x * lin_vel.x, dvm.y * lin_vel.y, dvm.z * lin_vel.z), vam = mk3(dvi.x * ang_vel.x, dvi.y * ang_vel.y, dvi.z * ang_vel.z);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        B00[3 * r + c] += sk(vam, r, c) - sk(ang_vel, r, c) * fl_comp(dvi, c);
        B01[3 * r + c] += sk(vlm, r, c) - sk(lin_vel, r, c) * fl_comp(dvm, c);
        B10[3 * r + c] += sk(vlm, r, c);
        B11[3 * r + c] += -sk(ang_vel, r, c) * fl_comp(dvm, c);
      }
  }
  const float blunt = fl[1], slender = fl[2], angdrag = fl[3], kutta = fl[4], magnus = fl[5];
  // Magnus
  const float volume = (float)(4.0 / 3.0 * 3.14159265358979323846) * s.x * s.y * s.z;
  const float magnus_coef = magnus * density * volume;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) { B10[3 * r + c] -= sk(lin_vel, r, c) * magnus_coef; B11[3 * r + c] += sk(ang_vel, r, c) * magnus_coef; }
  // Kutta lift
  const float a = (s.y * s.z) * (s.y * s.z), bb_ = (s.z * s.x) * (s.z * s.x), c = (s.x * s.y) * (s.x * s.y);
  const float aa = a * a, bb = bb_ * bb_, cc = c * c;
  const float x = lin_vel.x, y = lin_vel.y, z = lin_vel.z;
  const float xx = x * x, yy = y * y, zz = z * z;
  const float proj_denom = aa * xx + bb * yy + cc * zz, proj_num = a * xx + bb_ * yy + c * zz, norm2 = xx + yy + zz;
  const float df_denom = PI * kutta * density / fmaxf(MJ_MINVAL, sqrtf(proj_denom * proj_num * norm2));
  const v3 df = mk3(yy * (a - bb_) + zz * (a - c), xx * (bb_ - a) + zz * (bb_ - c), xx * (c - a) + yy * (c - bb_));
  const float proj_term = proj_num / fmaxf(MJ_MINVAL, proj_denom), cos_term = proj_num / fmaxf(MJ_MINVAL, norm2);
  const v3 sv = mk3(bb_ - c, c - a, a - bb_);
  const v3 inner_term = mk3(aa * proj_term - a + cos_term, bb * proj_term - bb_ + cos_term, cc * proj_term - c + cos_term);
  for (int r = 0; r < 3; r++)
    for (int q = 0; q < 3; q++) {
      float D = sk(sv, r, q) * (2.0f * proj_num) + fl_comp(df, r) * fl_comp(inner_term, q);
      D = fl_comp(lin_vel, r) * D * fl_comp(lin_vel, q) - (r == q ? fl_comp(df, r) * proj_num : 0.f);
      B11[3 * r + q] += D * df_denom;
    }
  // viscous drag
  const float d_max = fmaxf(fmaxf(s.x, s.y), s.z), d_min = fminf(fminf(s.x, s.y), s.z);
  const float d_mid = s.x + s.y + s.z - d_max - d_min;
  const float eq_sphere_D = (float)(2.0 / 3.0) * (s.x + s.y + s.z);
  const float A_max = PI * d_max * d_mid;
  const float A_proj = PI * sqrtf(proj_denom / fmaxf(MJ_MINVAL, proj_num));
  const float norm = sqrtf(xx + yy + zz), inv_norm = 1.0f / fmaxf(MJ_MINVAL, norm);
  const float lin_coef = viscosity * (float)(3.0 * 3.14159265358979323846) * eq_sphere_D;
  const float quad_coef = density * (A_proj * blunt + slender * (A_max - A_proj));
  const float Aproj_coef = density * norm * (blunt - slender);
  const float dA_coef = PI / fmaxf(MJ_MINVAL, sqrtf(proj_num * proj_num * proj_num * proj_denom));
  const v3 dAproj = mk3(Aproj_coef * dA_coef * a * x * (bb_ * yy * (a - bb_) + c * zz * (a - c)),
                        Aproj_coef * dA_coef * bb_ * y * (a * xx * (bb_ - a) + c * zz * (bb_ - c)),
                        Aproj_coef * dA_coef * c * z * (a * xx * (c - a) + bb_ * yy * (c - bb_)));
  const float inner = dot(lin_vel, lin_vel);
  for (int r = 0; r < 3; r++)
    for (int q = 0; q < 3; q++) {
      float D = (fl_comp(lin_vel, r) * fl_comp(lin_vel, q) + (r == q ? inner : 0.f)) * (-quad_coef * inv_norm);
      D -= fl_comp(lin_vel, r) * fl_comp(dAproj, q);
      D -= r == q ? lin_coef : 0.f;
      B11[3 * r + q] += D;
    }
  // viscous torque
  const float lin_visc_torq_coef = PI * eq_sphere_D * eq_sphere_D * eq_sphere_D;
  const float I_max = (float)(8.0 / 15.0 * 3.14159265358979323846) * d_mid * d_max * d_max * d_max * d_max;
  const v3 II = mk3(fluid_max_moment(s, 0), fluid_max_moment(s, 1), fluid_max_moment(s, 2));
  const v3 mom_coef = mk3(angdrag * II.x + slender * (I_max - II.x), angdrag * II.y + slender * (I_max - II.y), angdrag * II.z + slender * (I_max - II.z));
  const v3 mom_visc = mk3(ang_vel.x * mom_coef.x, ang_vel.y * mom_coef.y, ang_vel.z * mom_coef.z);
  const float density_scaled = density / fmaxf(MJ_MINVAL, length(mom_visc));
  const v3 mom_sq = mk3(-density_scaled * (ang_vel.x * mom_coef.x) * mom_coef.x, -density_scaled * (ang_vel.y * mom_coef.y) * mom_coef.y,
                        -density_scaled * (ang_vel.z * mom_coef.z) * mom_coef.z);
  const float diag_val = dot(ang_vel, mom_sq) - viscosity * lin_visc_torq_coef;
  for (int r = 0; r < 3; r++)
    for (int q = 0; q < 3; q++) B00[3 * r + q] += fl_comp(ang_vel, r) * fl_comp(mom_sq, q) + (r == q ? diag_val : 0.f);
  if constexpr (SYM) {
  // symmetrize (implicitfast) into B
  for (int r = 0; r < 3; r++)
    for (int q = 0; q < 3; q++) {
      const float b01 = 0.5f * (B01[3 * r + q] + B10[3 * q + r]);
      B[6 * r + q] = 0.5f * (B00[3 * r + q] + B00[3 * q + r]);
      B[6 * (r + 3) + q + 3] = 0.5f * (B11[3 * r + q] + B11[3 * q + r]);
      B[6 * r + q + 3] = b01;
      B[6 * (q + 3) + r] = b01;
    }
  } else {
    for (int r = 0; r < 3; r++)
      for (int q = 0; q < 3; q++) {
        B[6 * r + q] = B00[3 * r + q];
        B[6 * r + q + 3] = B01[3 * r + q];
        B[6 * (r + 3) + q] = B10[3 * r + q];
        B[6 * (r + 3) + q + 3] = B11[3 * r + q];
      }
  }
}

// The local Jacobian column of dof dd at a point with offset `off` from the subtree root's com, in the frame R: [R^T ang; R^T lin].
static __device__ __forceinline__ void fluid_jac_local(const float* cdof, v3 off, const float* R, float* J) {
  const v3 ang = ld3(cdof);
  const v3 jp = ld3(cdof + 3) + cross(ang, off);
  st3(J, fl_mtv(R, ang)); st3(J + 3, fl_mtv(R, jp));
}
