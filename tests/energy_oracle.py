"""fp64 numpy restatement of the reference's energy terms (sensor.py:2773-3019), per world.

potential: -sum_{b >= 1} body_mass[b] gravity . xipos[b] (unless gravity is disabled), plus 1/2 k x^2 for every joint spring (hinge /
slide: q - qpos_spring; ball: |quat_sub(normalize(q), q_spring)|; free: the translation and the rotation, each as its own term) and
every fixed-tendon spring (x: the length outside the dead band tendon_lengthspring = [lower, upper]) unless springs are disabled.
kinetic: 1/2 qvel . M qvel with M the world's lower triangle in MuJoCo's compressed layout (M_rowadr / M_colind).
"""
import numpy as np

from mujoco_warp_b200._src import constants as C


def quat_sub_length(q, q_spring):
  q = np.asarray(q, dtype=np.float64)
  q = q / np.linalg.norm(q)
  a, b = np.array([q_spring[0], -q_spring[1], -q_spring[2], -q_spring[3]]), q
  qd = np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                 a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])
  s = np.linalg.norm(qd[1:])
  if s == 0.0:
    return 0.0
  speed = 2.0 * np.arctan2(s, qd[0])
  if speed > np.pi:
    speed -= 2.0 * np.pi
  return float(np.linalg.norm(qd[1:] * speed / s))


def field(mjm, inputs, name, w):
  """world w's value of a Model field: the per-world input if the scene randomises it, else the model's"""
  return np.asarray(inputs[name][w] if name in inputs else getattr(mjm, name), dtype=np.float64)


def potential_terms(mjm, inputs, w, qpos, xipos, ten_length):
  """(gravity terms, spring terms) of world w as arrays, so that callers can also scale tolerances by sum |term|"""
  dis = int(mjm.opt.disableflags)
  grav, spring = [], []
  if not dis & C.DSBL_GRAVITY:
    mass, g = field(mjm, inputs, "body_mass", w), np.asarray(mjm.opt.gravity, dtype=np.float64)
    grav = [-mass[b] * float(g @ xipos[b]) for b in range(1, mjm.nbody)]
  if not dis & C.DSBL_SPRING:
    k, qs = field(mjm, inputs, "jnt_stiffness", w), field(mjm, inputs, "qpos_spring", w)
    for j in range(mjm.njnt):
      if k[j] == 0.0:
        continue
      a, t = int(mjm.jnt_qposadr[j]), int(mjm.jnt_type[j])
      if t == C.JNT_FREE:
        spring += [0.5 * k[j] * float(np.sum((qpos[a : a + 3] - qs[a : a + 3]) ** 2)), 0.5 * k[j] * quat_sub_length(qpos[a + 3 : a + 7], qs[a + 3 : a + 7]) ** 2]
      elif t == C.JNT_BALL:
        spring.append(0.5 * k[j] * quat_sub_length(qpos[a : a + 4], qs[a : a + 4]) ** 2)
      else:
        spring.append(0.5 * k[j] * (qpos[a] - qs[a]) ** 2)
    nt = int(getattr(mjm, "ntendon", 0))
    if nt:
      kt, ls = field(mjm, inputs, "tendon_stiffness", w), field(mjm, inputs, "tendon_lengthspring", w).reshape(nt, 2)
      for t in range(nt):
        if kt[t] == 0.0:
          continue
        L, lo, hi = ten_length[t], ls[t, 0], ls[t, 1]
        x = L - hi if L > hi else (L - lo if L < lo else 0.0)
        spring.append(0.5 * kt[t] * x * x)
  return np.asarray(grav, dtype=np.float64), np.asarray(spring, dtype=np.float64)


def dense_m(mjm, M):
  from mujoco_warp_b200._src import io as mio

  row = mio.derive_tables(mjm)["M_entry_row"]
  out = np.zeros((mjm.nv, mjm.nv))
  for e, (i, j) in enumerate(zip(row, np.asarray(mjm.M_colind))):
    out[i, j] = out[j, i] = M[e]
  return out


def kinetic_terms(mjm, qvel, M):
  """the products qvel_i M_ij qvel_j / 2 whose sum is the kinetic energy"""
  return 0.5 * np.outer(qvel, qvel) * dense_m(mjm, M)


def energy(mjm, inputs, g, w):
  """(potential, kinetic) of world w from a fixture's forward state"""
  grav, spring = potential_terms(mjm, inputs, w, g["in/qpos"][w], g["forward/xipos"][w], g["forward/ten_length"][w])
  return float(grav.sum() + spring.sum()), float(kinetic_terms(mjm, g["in/qvel"][w], g["forward/M"][w]).sum())
