"""Scenes for the magnetometer, camprojection, insidesite, tendon limit and tendonactfrc sensors (tests/test_sensor_extra_host.py,
tests/test_gpu_sensor_extra.py, tools/make_sensor_extra_goldens.py, tools/sensor_extra_bench.py).

One model carries every case:
- a two-link arm on hinges and a sled on a slide joint, with sites that move; a magnetometer on each (appended to the compiled arrays,
  MAGNETOMETERS: the MJCF compiler keeps refusing <magnetometer>);
- three cameras: a fixed one on the fovy path, a fixed one with focal length / sensor size (the intrinsic path) and one riding the arm;
  camprojection of the moving sites into each;
- a limited fixed tendon on the arm whose range is narrow enough that its limit row is active in most worlds, driven by two motors,
  and a limited tendon on the sled whose range is never reached (its limit sensors read 0), driven by one; limit pos / vel / frc and
  tendonactfrc on both;
- five static sites, one of each volume shape, each with a body, xbody, geom, site and camera object of its own (its frame origin
  and camera lie inside, its centre of mass, geom and site outside; INSIDE) and a massless body whose subtree com lies inside the sphere
  while its frame origin does not.  These objects do not move, so every tested point stays at least 0.05 from every site surface and
  insidesite is decided the same way in fp32 and fp64;
- cutoff on one sensor of each kind, and delayed sensors (a history of 3 samples).
`all_<integrator>` runs it with Euler, implicitfast and RK4; `batched` sets per-world opt.magnetic, cam_fovy and cam_intrinsic
(BATCHED); `alone_<tag>` keeps one sensor of one type.  Worlds start from seeded per-world qpos / qvel and take a seeded ctrl each step.
"""
import numpy as np

NWORLD = 3

# site shapes: name, type, size, position, euler (degrees)
SHAPES = (
  ("sph", "sphere", "0.3", (2.0, 0.0, 1.0), "0 0 0"),
  ("cap", "capsule", "0.2 0.3", (2.0, 1.2, 1.0), "30 0 20"),
  ("ell", "ellipsoid", "0.3 0.25 0.4", (2.0, 2.4, 1.0), "0 40 0"),
  ("cyl", "cylinder", "0.25 0.3", (2.0, 3.6, 1.0), "20 10 0"),
  ("box", "box", "0.2 0.3 0.35", (2.0, 4.8, 1.0), "15 25 35"),
)
# each shape's objects: a static body at the shape's centre + INSIDE (its frame origin is inside: xbody, and its camera sits there
# too), whose geom (and so its centre of mass, body) is 0.85 away along x and whose own site is 0.9 away along z (outside)
INSIDE = (0.05, 0.02, 0.03)


def _targets():
  out = []
  for name, typ, size, pos, euler in SHAPES:
    out.append(f'<site name="s_{name}" type="{typ}" size="{size}" pos="{pos[0]} {pos[1]} {pos[2]}" euler="{euler}"/>')
    p = np.asarray(pos) + INSIDE
    out.append(f'<body name="p_{name}" pos="{p[0]} {p[1]} {p[2]}"><geom name="g_{name}" type="sphere" size="0.05" pos="0.85 0 0" mass="1"/>'
               f'<site name="q_{name}" pos="0 0 0.9" size="0.01"/><camera name="c_{name}" pos="0.02 0 0"/></body>')
  # massless body 2 above the sphere site, with a massive child whose com (and so the subtree com) lies inside it
  out.append('<body name="massless" pos="2 0 3"><body name="massless_child" pos="0.05 0.05 -1.95"><geom type="sphere" size="0.02" mass="0.5"/></body></body>')
  return "\n    ".join(out)


def _inside_sensors(cutoff=False):
  out = []
  for name, *_ in SHAPES:
    for objtype, objname in (("body", f"p_{name}"), ("xbody", f"p_{name}"), ("geom", f"g_{name}"), ("site", f"q_{name}"), ("camera", f"c_{name}")):
      out.append(f'<insidesite objtype="{objtype}" objname="{objname}" site="s_{name}"/>')
  out.append('<insidesite objtype="body" objname="massless" site="s_sph"/>')
  out.append('<insidesite objtype="xbody" objname="massless" site="s_sph"/>')
  if cutoff:
    out.append('<insidesite objtype="xbody" objname="p_sph" site="s_sph" cutoff="0.5"/>')
  return out


ALL_SENSORS = [
  '<camprojection site="tip" camera="cam_fovy"/>', '<camprojection site="sled_s" camera="cam_intr"/>', '<camprojection site="sled_s" camera="cam_arm"/>',
  '<camprojection site="tip" camera="cam_intr" cutoff="150"/>',
  '<tendonlimitpos tendon="t_lim"/>', '<tendonlimitvel tendon="t_lim"/>', '<tendonlimitfrc tendon="t_lim"/>',
  '<tendonlimitpos tendon="t_free"/>', '<tendonlimitvel tendon="t_free"/>', '<tendonlimitfrc tendon="t_free"/>',
  '<tendonlimitfrc tendon="t_lim" cutoff="0.5"/>', '<tendonactfrc tendon="t_lim"/>', '<tendonactfrc tendon="t_free"/>',
  '<tendonactfrc tendon="t_lim" cutoff="0.3"/>',
  # delayed (3-sample history) sensors of each stage
  '<camprojection site="tip" camera="cam_arm" nsample="3" delay="0.003"/>', '<tendonlimitvel tendon="t_lim" nsample="3" delay="0.002"/>',
  '<tendonactfrc tendon="t_lim" nsample="3" delay="0.004"/>',
  # sensors this build already carried, next to the new ones
  '<jointpos joint="j1"/>', '<tendonpos tendon="t_lim"/>',
] + _inside_sensors(cutoff=True)

# magnetometers (site, cutoff, nsample, delay), appended to the compiled arrays: the MJCF compiler keeps refusing <magnetometer>, and
# put_model runs those a model carries in its arrays
MAGNETOMETERS = (("tip", 0.0, 0, 0.0), ("sled_s", 0.0, 0, 0.0), ("tip", 0.2, 0, 0.0), ("tip", 0.0, 3, 0.003))

ALONE = {
  "magnetometer": None, "camprojection": '<camprojection site="tip" camera="cam_fovy"/>',
  "insidesite": '<insidesite objtype="xbody" objname="p_box" site="s_box"/>', "tendonlimitpos": '<tendonlimitpos tendon="t_lim"/>',
  "tendonlimitvel": '<tendonlimitvel tendon="t_lim"/>', "tendonlimitfrc": '<tendonlimitfrc tendon="t_lim"/>', "tendonactfrc": '<tendonactfrc tendon="t_lim"/>',
}

XML = """
<mujoco model="sensor_extra">
  <option timestep="0.002" integrator="{integrator}" magnetic="0.1 -0.4 0.25"/>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <camera name="cam_fovy" pos="0 -3 1" xyaxes="1 0 0 0 0 1" fovy="50" resolution="640 480"/>
    <camera name="cam_intr" pos="0.3 -3 1.5" xyaxes="1 0 0 0 0.2 1" resolution="320 240" sensorsize="0.0048 0.0036" focal="0.004 0.0045"/>
    <body name="arm" pos="0 0 1">
      <joint name="j1" type="hinge" axis="0 1 0" damping="0.1"/>
      <geom type="capsule" fromto="0 0 0 0.4 0 0" size="0.03" mass="0.8"/>
      <camera name="cam_arm" pos="0.2 -0.5 0.1" xyaxes="1 0 0 0 0 1" fovy="70" resolution="200 100"/>
      <body name="fore" pos="0.4 0 0">
        <joint name="j2" type="hinge" axis="0 1 0" damping="0.05"/>
        <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.02" mass="0.4"/>
        <site name="tip" pos="0.3 0 0" size="0.01"/>
      </body>
    </body>
    <body name="sled" pos="0 1 0.5">
      <joint name="slide" type="slide" axis="1 0 0" damping="0.3"/>
      <geom type="box" size="0.05 0.05 0.05" mass="1.0"/>
      <site name="sled_s" pos="0 0 0.1" euler="10 20 30" size="0.01"/>
    </body>
    {targets}
  </worldbody>
  <tendon>
    <fixed name="t_lim" limited="true" range="-0.04 0.05" margin="0.01">
      <joint joint="j1" coef="1"/>
      <joint joint="j2" coef="0.5"/>
    </fixed>
    <fixed name="t_free" limited="true" range="-50 50">
      <joint joint="slide" coef="1"/>
    </fixed>
  </tendon>
  <actuator>
    <motor name="m_lim_a" tendon="t_lim" gear="2"/>
    <motor name="m_j2" joint="j2" gear="0.5"/>
    <motor name="m_lim_b" tendon="t_lim" gear="-0.7"/>
    <motor name="m_free" tendon="t_free" gear="1.5"/>
  </actuator>
  <sensor>
    {sensors}
  </sensor>
</mujoco>"""


def xml(integrator="Euler", sensors=None):
  return XML.format(integrator=integrator, targets=_targets(), sensors="\n    ".join(ALL_SENSORS if sensors is None else sensors))


def add_magnetometers(m, mags):
  """Appends magnetometers (site name, cutoff, nsample, delay) to a compiled model's sensor arrays, as MuJoCo's compiler lays them out."""
  from mujoco_warp_b200._src import constants as C
  from mujoco_warp_b200._src import mjcf

  for site, cutoff, nsample, delay in mags:
    row = dict(type=C.SENS_MAGNETOMETER, objtype=C.OBJ_SITE, objid=list(m.names.site).index(site), reftype=C.OBJ_UNKNOWN, refid=-1, dim=3, datatype=0, needstage=1)
    for k, v in row.items():
      setattr(m, "sensor_" + k, np.append(np.asarray(getattr(m, "sensor_" + k)), v).astype(np.int32))
    m.sensor_adr = np.append(m.sensor_adr, m.nsensordata).astype(np.int32)
    m.sensor_intprm = np.concatenate([np.asarray(m.sensor_intprm).reshape(-1, 3), np.zeros((1, 3), dtype=np.int32)])
    m.sensor_cutoff, m.sensor_noise = np.append(m.sensor_cutoff, cutoff), np.append(m.sensor_noise, 0.0)
    m.sensor_history = np.concatenate([np.asarray(m.sensor_history).reshape(-1, 2), np.array([[nsample, 0]], dtype=np.int32)])
    m.sensor_delay = np.append(m.sensor_delay, delay)
    m.sensor_interval = np.concatenate([np.asarray(m.sensor_interval).reshape(-1, 2), np.zeros((1, 2))])
    m.names.sensor = list(m.names.sensor) + [f"magnetometer{m.nsensor}"]
    m.nsensor += 1
    m.nsensordata += 3
  mjcf.set_history_layout(m)
  return m


def _load(integrator="Euler", sensors=None, mags=MAGNETOMETERS):
  from mujoco_warp_b200._src import mjcf

  return add_magnetometers(mjcf.load_string(xml(integrator, sensors)), mags)


# name: (model source, steps, per-world fields)
SCENES = {
  "all_euler": (lambda: _load("Euler"), 8, False),
  "all_implicitfast": (lambda: _load("implicitfast"), 6, False),
  "all_rk4": (lambda: _load("RK4"), 5, False),
  "batched": (lambda: _load("Euler"), 5, True),
  "alone_magnetometer": (lambda: _load("Euler", [], MAGNETOMETERS[:1]), 4, False),
  **{f"alone_{k}": ((lambda s: lambda: _load("Euler", [s], ()))(v), 4, False) for k, v in ALONE.items() if v},
}


def load(name):
  return SCENES[name][0]()


def batched(mjm, nworld=NWORLD):
  """Per-world opt.magnetic (nworld, 3), cam_fovy (nworld, ncam) and cam_intrinsic (nworld, ncam, 4)."""
  k = np.arange(nworld, dtype=np.float64)
  mag = np.asarray(mjm.opt.magnetic, dtype=np.float64)[None] * (1.0 + 0.5 * k[:, None]) + np.stack([0.1 * k, -0.05 * k, 0.2 * k], axis=1)
  fovy = np.asarray(mjm.cam_fovy, dtype=np.float64)[None] + 7.5 * k[:, None]
  intr = np.asarray(mjm.cam_intrinsic, dtype=np.float64)[None] * (1.0 + 0.25 * k[:, None, None])
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(mag), f32(fovy), f32(intr)


def seeded(mjm, nsteps, nworld=NWORLD, seed=11):
  """Per-world qpos / qvel and a per-world, per-step ctrl (nsteps, nworld, nu), fp32-representable."""
  from tests import util

  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=None, seed=seed, qpos_noise=0.1, qvel_noise=0.5, exact_world0=False)
  rng = np.random.default_rng(seed)
  ctrl = rng.uniform(-1.0, 1.0, (nsteps, nworld, int(mjm.nu)))
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel), f32(ctrl)
