// k_integrate.cu -- Euler (+ optional implicit joint damping) and implicitfast integrators, harness ctrl-noise kernel.
//
// Replaces (reference, /root/reference/mujoco_warp/_src/): forward.py:387-417 euler, :276-349 _advance
// (_next_velocity :117, _next_position :53, _next_time :221, qacc_warmstart copy :343) and, for models without
// eulerdamp=disable, the (M + dt*diag(damping)) factor-solve (:391-415).  implicitfast (forward.py:602-610 with
// derivative.py:38-176 _qderiv_actuator_passive_vel, :178-245 moment^T vel moment scatter, :221-245 damping) factors
// M - dt*qDeriv instead.  cli.py:103-145 _ctrl_noise.
#include "mjb_chol.cuh"
#include "mjb_implicit_a.cuh"
#include "mjb_launch.cuh"
#include "mjb_math.cuh"
#include "mjb_types.cuh"

namespace {

__host__ __device__ inline int chol_ld(int n) { return (n | 1); }
__host__ __device__ inline int int_words(const ModelDev& m) {
  const bool damp = m.integrator == INT_IMPLICITFAST || !(m.disableflags & (DSBL_EULERDAMP | DSBL_DAMPER));
  int o = 2 * m.nv;  // qacc, qvel
  if (damp) o += m.maxtree * chol_ld(m.maxtree) + m.maxtree;
  return (o + 3) & ~3;
}

// FLUID: implicitfast includes the fluid force derivatives (k_euler_fluid)
template <bool FLUID, bool BAT>
__device__ __forceinline__ void euler(const ModelDev& mp, const DataDev& d, int integrator, const FluidDev& f) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x, warp = 0;  // one warp per block: the world index is block-uniform
  const int w = blockIdx.x + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  float* S = smem + warp * int_words(mp);
  float *qacc = S, *qvel = S + m.nv, *A = S + 2 * m.nv, *x = A + m.maxtree * chol_ld(m.maxtree);
  const int nv = m.nv;
  const size_t wb = (size_t)w;
  const float dt = m.timestep;

  warp_copy(qacc, d.qacc + wb * nv, nv, lane);
  warp_copy(qvel, d.qvel + wb * nv, nv, lane);
  __syncwarp();
  warp_copy(d.qacc_warmstart + wb * nv, qacc, nv, lane);  // warmstart <- solver qacc (forward.py:343)

  const bool implicitfast = integrator == INT_IMPLICITFAST;
  if (integrator == INT_IMPLICIT) {  // forward.py:578-600: the acceleration k_implicit solved for with the full velocity derivative
    __syncwarp();
    warp_copy(qacc, d.imp_qacc + wb * nv, nv, lane);
    __syncwarp();
  } else if (implicitfast || !(m.disableflags & (DSBL_EULERDAMP | DSBL_DAMPER))) {
    // Euler: qacc <- (M + dt*diag(damping))^-1 * Ma  (forward.py:391-415); implicitfast: (M - dt*qDeriv)^-1 * Ma
    const bool damper = !(m.disableflags & DSBL_DAMPER);
    const float* Mw = d.M + wb * m.nC;
#pragma unroll 1
    for (int t = 0; t < m.ntree; t++) {
      const int start = m.tree_dofadr[t], n = m.tree_dofnum[t], ld = chol_ld(n);
      tree_implicit_a<FLUID>(m, d, wb, Mw, start, n, ld, dt, implicitfast, damper, A, lane, f);
      if (n <= 32) {
        const float b = lane < n ? d.efc_Ma[wb * nv + start + lane] : 0.f;
        const float xx = chol_solve_reg_any(A, ld, n, b, A, ld, lane);
        if (lane < n) x[lane] = xx;
        __syncwarp();
      } else {
#pragma unroll 1
        for (int i = lane; i < n; i += 32) x[i] = d.efc_Ma[wb * nv + start + i];
        __syncwarp();
        warp_cholesky(A, n, ld, lane);
        warp_chol_solve(A, n, ld, x, lane);
      }
#pragma unroll 1
      for (int i = lane; i < n; i += 32) qacc[start + i] = x[i];
      __syncwarp();
    }
  }
#pragma unroll 1
  for (int dd = lane; dd < nv; dd += 32) { const float v = qvel[dd] + qacc[dd] * dt; qvel[dd] = v; d.qvel[wb * nv + dd] = v; }
  __syncwarp();
  float* qpos = d.qpos + wb * m.nq;
#pragma unroll 1
  for (int j = lane; j < m.njnt; j += 32) {
    const int t = m.jnt_type[j], qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
    if (t == JNT_FREE) {
      for (int k = 0; k < 3; k++) qpos[qa + k] += dt * qvel[da + k];
      stq(qpos + qa + 3, quat_integrate(ldq(qpos + qa + 3), ld3(qvel + da + 3), dt));
    } else if (t == JNT_BALL) {
      stq(qpos + qa, quat_integrate(ldq(qpos + qa), ld3(qvel + da), dt));
    } else {
      qpos[qa] += dt * qvel[da];
    }
  }
  if (lane == 0) {  // _next_time (forward.py:221-271)
    d.time[w] += dt;
    int ovf = 0;
    if (d.nefc[w] > d.njmax) ovf |= OVF_NEFC;
    if (d.ncollision[0] > d.naconmax) ovf |= OVF_BROADPHASE;
    if (d.nacon[0] > d.naconmax) ovf |= OVF_NARROWPHASE;
    if (ovf) d.overflow[w] |= ovf;
  }
}

template <bool BAT>
__global__ void __launch_bounds__(32)
k_euler(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int integrator) { euler<false, BAT>(mp, d, integrator, FluidDev{}); }
template <bool BAT>
__global__ void __launch_bounds__(32)
k_euler_fluid(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, int integrator, const __grid_constant__ FluidDev f) {
  euler<true, BAT>(mp, d, integrator, f);
}

// deterministic Halton value (reference util_misc.py:61-76)
__device__ __forceinline__ float halton(int index, int base) {
  int n0 = index;
  const float b = (float)base;
  float f = 1.0f / b, hn = 0.f;
  while (n0 > 0) { const int n1 = n0 / base, r = n0 - n1 * base; hn += f * (float)r; f /= b; n0 = n1; }
  return hn;
}

template <bool BAT>
__global__ void k_ctrl_noise(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, const float* __restrict__ ctrl_center, int step, float noise_std, float noise_rate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.nworld * mp.nu) return;
  const int w = i / mp.nu, a = i - w * mp.nu;
  MJB_WORLD_MODEL(w)
  const float rate = expf(-m.timestep / noise_rate), scale = noise_std * sqrtf(1.0f - rate * rate);
  float midpoint = 0.f, halfrange = 1.f;
  const float lo = m.actuator_ctrlrange[2 * a], hi = m.actuator_ctrlrange[2 * a + 1];
  const bool limited = m.actuator_ctrllimited[a];
  if (limited) { midpoint = 0.5f * (hi + lo); halfrange = 0.5f * (hi - lo); }
  if (ctrl_center) midpoint = ctrl_center[a];
  float ctrl = rate * d.ctrl[i] + (1.0f - rate) * midpoint;
  ctrl += scale * halfrange * (2.0f * halton((step + 1) * (w + 1), a + 2) - 1.0f);
  if (limited) ctrl = clampf(ctrl, lo, hi);
  d.ctrl[i] = ctrl;
}

// forward.py:53-115 _next_position for one joint: qpos <- integrate(qpos_in, scale * qvel) over dt
__device__ __forceinline__ void next_position_jnt(const ModelDev& m, int j, const float* qpos_in, const float* qvel, float scale, float dt, float* qpos) {
  const int t = m.jnt_type[j], qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
  if (t == JNT_FREE) {
    for (int k = 0; k < 3; k++) qpos[qa + k] = qpos_in[qa + k] + dt * (qvel[da + k] * scale);
    stq(qpos + qa + 3, quat_integrate(ldq(qpos_in + qa + 3), ld3(qvel + da + 3) * scale, dt));
  } else if (t == JNT_BALL) {
    stq(qpos + qa, quat_integrate(ldq(qpos_in + qa), ld3(qvel + da) * scale, dt));
  } else {
    qpos[qa] = qpos_in[qa] + dt * qvel[da] * scale;
  }
}

// Plain Euler without the implicit-damping solve (eulerdamp disabled or no dampers: the benchmark humanoid): nothing couples
// the dofs, so the stage is an elementwise pass -- one THREAD per (world, joint) advances the joint's velocities, warm start
// and position (forward.py:276-349 _advance); consecutive threads touch consecutive addresses, no shared memory, and the
// grid is sized by joints instead of worlds.  k_euler (one warp per world) remains for the factor-and-solve variants.
__global__ void __launch_bounds__(256)
k_euler_flat(const __grid_constant__ ModelDev m, const __grid_constant__ DataDev d) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int wl = idx / m.njnt, j = idx - wl * m.njnt;
  if (wl >= d.wn) return;
  const int w = wl + d.w0;
  if (w >= d.nworld) return;
  const size_t wb = (size_t)w;
  const float dt = m.timestep;
  const int t = m.jnt_type[j], qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
  const int nd = t == JNT_FREE ? 6 : (t == JNT_BALL ? 3 : 1);
  float v[6];
#pragma unroll
  for (int k = 0; k < 6; k++) {
    if (k < nd) {
      const float a = d.qacc[wb * m.nv + da + k];
      v[k] = d.qvel[wb * m.nv + da + k] + a * dt;
      d.qvel[wb * m.nv + da + k] = v[k];
      d.qacc_warmstart[wb * m.nv + da + k] = a;  // warmstart <- solver qacc (forward.py:343)
    }
  }
  float* qpos = d.qpos + wb * m.nq;
  if (t == JNT_FREE) {
    for (int k = 0; k < 3; k++) qpos[qa + k] += dt * v[k];
    stq(qpos + qa + 3, quat_integrate(ldq(qpos + qa + 3), mk3(v[3], v[4], v[5]), dt));
  } else if (t == JNT_BALL) {
    stq(qpos + qa, quat_integrate(ldq(qpos + qa), mk3(v[0], v[1], v[2]), dt));
  } else {
    qpos[qa] += dt * v[0];
  }
  if (j == 0) {  // _next_time (forward.py:221-271)
    d.time[w] += dt;
    int ovf = 0;
    if (d.nefc[w] > d.njmax) ovf |= OVF_NEFC;
    if (d.ncollision[0] > d.naconmax) ovf |= OVF_BROADPHASE;
    if (d.nacon[0] > d.naconmax) ovf |= OVF_NARROWPHASE;
    if (ovf) d.overflow[w] |= ovf;
  }
}

// forward.py:135-218 _next_activation (dyntype NONE / INTEGRATOR / FILTER / FILTEREXACT): one thread per (world, actuator)
// advances the actuator's activations from act_dot; launched after the integrator kernel (which still reads the old ones).
template <bool BAT>
__global__ void __launch_bounds__(256)
k_next_act(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int wl = idx / mp.nu, a = idx - wl * mp.nu;
  if (wl >= d.wn) return;
  const int w = wl + d.w0;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const int adr = m.actuator_actadr[a];
  if (adr < 0) return;
  for (int j = adr; j < adr + m.actuator_actnum[a]; j++) {
    const size_t k = (size_t)w * m.na + j;
    d.act[k] = next_act(m, a, d.act[k], d.act_dot[k], 1.0f, m.actuator_actlimited[a] != 0);
  }
}

// One Runge-Kutta bookkeeping step after the stage-th forward() of the step (forward.py:523-555 rungekutta4, stateless
// actuators): accumulate B[stage] * (qvel, qacc); stages 0..2 then perturb the state for the next forward
// (_rk_perturb_state: position from the current stage velocity, velocity from qvel_t0 + A dt qacc); stage 3 restores the
// state and advances it with the accumulated velocity / acceleration (_advance with qvel = qvel_rk).
// rk: per world [qpos_t0 (nq) | qvel_t0 (nv) | qvel_rk (nv) | qacc_rk (nv) | act_t0 (na) | act_dot_rk (na)].  One warp per world.
// Stateful actuators (forward.py:445-463, 514-519, 553-555): stage activations are next_act(act_t0, act_dot, A) without the range
// clamp, the final ones next_act(act_t0, sum B act_dot, 1) with it.
template <bool BAT>
__global__ void __launch_bounds__(32)
k_rk_stage(const __grid_constant__ ModelDev mp, const __grid_constant__ DataDev d, float* __restrict__ rk, int stage) {
  const int lane = threadIdx.x, w = blockIdx.x;
  if (w >= d.nworld) return;
  MJB_WORLD_MODEL(w)
  const int nq = m.nq, nv = m.nv;
  const size_t wb = (size_t)w;
  const int na = m.na;
  float *qpos_t0 = rk + wb * (nq + 3 * nv + 2 * na), *qvel_t0 = qpos_t0 + nq, *qvel_rk = qvel_t0 + nv, *qacc_rk = qvel_rk + nv, *act_t0 = qacc_rk + nv, *act_dot_rk = act_t0 + na;
  float *act = d.act + wb * na, *act_dot = d.act_dot + wb * na;
  float *qpos = d.qpos + wb * nq, *qvel = d.qvel + wb * nv;
  const float* qacc = d.qacc + wb * nv;
  const float dt = m.timestep;
  const float B = (stage == 0 || stage == 3) ? (1.0f / 6.0f) : (1.0f / 3.0f), A = stage == 2 ? 1.0f : 0.5f;
  if (stage == 0) {
    for (int i = lane; i < nq; i += 32) qpos_t0[i] = qpos[i];
    for (int i = lane; i < nv; i += 32) { const float v = qvel[i]; qvel_t0[i] = v; qvel_rk[i] = B * v; qacc_rk[i] = B * qacc[i]; }
    for (int i = lane; i < na; i += 32) { act_t0[i] = act[i]; act_dot_rk[i] = B * act_dot[i]; }
  } else {
    for (int i = lane; i < nv; i += 32) { qvel_rk[i] += B * qvel[i]; qacc_rk[i] += B * qacc[i]; }
    for (int i = lane; i < na; i += 32) act_dot_rk[i] += B * act_dot[i];
  }
  __syncwarp();
  if (stage < 3) {
    for (int j = lane; j < m.njnt; j += 32) next_position_jnt(m, j, qpos_t0, qvel, A, dt, qpos);
    __syncwarp();
    for (int i = lane; i < nv; i += 32) qvel[i] = qvel_t0[i] + A * qacc[i] * dt;
    if (na > 0)
      for (int a = lane; a < m.nu; a += 32)
        for (int j = m.actuator_actadr[a]; j >= 0 && j < m.actuator_actadr[a] + m.actuator_actnum[a]; j++) act[j] = next_act(m, a, act_t0[j], act_dot[j], A, false);
    return;
  }
  if (na > 0) {
    for (int a = lane; a < m.nu; a += 32)
      for (int j = m.actuator_actadr[a]; j >= 0 && j < m.actuator_actadr[a] + m.actuator_actnum[a]; j++) {
        act_dot[j] = act_dot_rk[j];
        act[j] = next_act(m, a, act_t0[j], act_dot_rk[j], 1.0f, m.actuator_actlimited[a] != 0);
      }
  }
  for (int i = lane; i < nv; i += 32) { qvel[i] = qvel_t0[i] + qacc_rk[i] * dt; d.qacc_warmstart[wb * nv + i] = qacc[i]; }
  for (int j = lane; j < m.njnt; j += 32) next_position_jnt(m, j, qpos_t0, qvel_rk, 1.0f, dt, qpos);
  if (lane == 0) {  // _next_time (forward.py:221-271)
    d.time[w] += dt;
    int ovf = 0;
    if (d.nefc[w] > d.njmax) ovf |= OVF_NEFC;
    if (d.ncollision[0] > d.naconmax) ovf |= OVF_BROADPHASE;
    if (d.nacon[0] > d.naconmax) ovf |= OVF_NARROWPHASE;
    if (ovf) d.overflow[w] |= ovf;
  }
}


}  // namespace

size_t smem_integrate(const ModelDev& m) { return (size_t)int_words(m) * sizeof(float); }

// integrator: INT_EULER / INT_IMPLICITFAST / INT_IMPLICIT, or -1 for the model's own (RK4 models advance with Euler here, forward.py:1411)
cudaError_t launch_integrate(const ModelDev& m, const DataDev& d, int integrator, cudaStream_t s, const FluidDev& f) {
  if (integrator < 0) integrator = (m.integrator == INT_IMPLICITFAST || m.integrator == INT_IMPLICIT) ? m.integrator : INT_EULER;
  const bool solve = integrator == INT_IMPLICITFAST || integrator == INT_IMPLICIT || !(m.disableflags & (DSBL_EULERDAMP | DSBL_DAMPER));
  cudaError_t e = integrator == INT_IMPLICIT ? launch_implicit_solve(m, d, d.imp_qacc, s) : cudaSuccess;
  if (e != cudaSuccess) return e;
  if (!solve && m.njnt > 0) {
    const long n = (long)d.wn * m.njnt;
    e = launch(k_euler_flat, (unsigned)((n + 255) / 256), 256, 0, s, m, d);
  } else {
    e = f.has_fluid ? launch(m.batched ? k_euler_fluid<true> : k_euler_fluid<false>, d.wn, 32, smem_integrate(m), s, m, d, integrator, f)
                    : launch(m.batched ? k_euler<true> : k_euler<false>, d.wn, 32, smem_integrate(m), s, m, d, integrator);
  }
  if (e != cudaSuccess || m.na <= 0 || m.nu <= 0) return e;
  const long n = (long)d.wn * m.nu;  // after the integrator kernel: it reads the activations of the step
  return launch(m.batched ? k_next_act<true> : k_next_act<false>, (unsigned)((n + 255) / 256), 256, 0, s, m, d);
}

cudaError_t launch_ctrl_noise(const ModelDev& m, const DataDev& d, const float* ctrl_center, int step, float std, float rate, cudaStream_t s) {
  const int n = d.nworld * m.nu;
  if (n == 0) return cudaSuccess;
  return launch(m.batched ? k_ctrl_noise<true> : k_ctrl_noise<false>, (n + 255) / 256, 256, 0, s, m, d, ctrl_center, step, std, rate);
}

cudaError_t launch_rk_stage(const ModelDev& m, const DataDev& d, float* rk, int stage, cudaStream_t s) {
  return launch(m.batched ? k_rk_stage<true> : k_rk_stage<false>, d.nworld, 32, 0, s, m, d, rk, stage);
}
