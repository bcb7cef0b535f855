"""Scenes for the rangefinder sensor (tests/test_rangefinder_host.py, tests/test_gpu_rangefinder.py, tools/make_rangefinder_goldens.py).

The MJCF compiler keeps refusing <rangefinder>; `add_rangefinders` puts the sensors into a compiled model's arrays as MuJoCo's compiler lays
them out (type 7, a site object, one POSITIVE output, position stage), appended or inserted between the model's own sensors.

One model carries the primitive cases: a hinged arm and a sled on a slide joint, whose sites' z axes sweep over a floor and static
sphere / capsule / ellipsoid / cylinder / box geoms, and over moving geoms on each other.  Around them:
- a site whose own body has a geom in front of it (the sled's box below its centre site), a site on the world body (every world geom,
  floor included, is excluded from its ray) and a site on a static body inside a sphere of the world body;
- an alpha-0 geom, a geom with an alpha-0 material (both invisible to rays), a non-colliding visual geom and geoms in groups 3-5 (hit);
- rays that miss (pointing at the sky), cutoffs above and below the hit distance and on a miss.
No geom pair can collide (the moving geoms have contype = conaffinity = 0), so the worlds differ only by their seeded joint motion.
`mesh` aims sites at mesh faces; `delay` gives rangefinders nsample / delay / interval; `batched` sets per-world geom_size and geom_rgba
(alpha 0 in some worlds only); `many` carries a grid of 210 rangefinders; `<integrator>` runs the primitive scene with each integrator.
"""
import numpy as np

NWORLD = 3

XML = """
<mujoco model="rangefinder">
  <option timestep="0.002" integrator="{integrator}"/>
  <asset>
    <material name="ghost" rgba="1 1 1 0"/>
    <material name="red" rgba="1 0 0 1"/>
    {assets}
  </asset>
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <geom name="floor" type="plane" size="0 0 1" contype="1" conaffinity="1"/>
    <geom name="s_sphere" type="sphere" size="0.2" pos="0.6 0 0.25" contype="1" conaffinity="1"/>
    <geom name="s_capsule" type="capsule" size="0.08 0.25" pos="-0.6 0 0.3" euler="90 0 0" contype="1" conaffinity="1" group="3"/>
    <geom name="s_ellipsoid" type="ellipsoid" size="0.25 0.15 0.1" pos="0 0.6 0.3" euler="0 0 30" material="red" group="4"/>
    <geom name="s_cylinder" type="cylinder" size="0.15 0.1" pos="0 -0.6 0.3" euler="20 0 0" group="5"/>
    <geom name="s_box" type="box" size="0.2 0.15 0.1" pos="1.2 0 0.2" euler="0 0 25"/>
    <geom name="invisible" type="box" size="0.3 0.3 0.02" pos="0.3 0 0.6" rgba="1 1 1 0"/>
    <geom name="ghost" type="box" size="0.3 0.3 0.02" pos="-0.3 0 0.6" material="ghost"/>
    <geom name="visual" type="box" size="0.1 0.3 0.02" pos="0 0 0.55" group="3"/>
    <geom name="big" type="sphere" size="0.3" pos="2 2 1"/>
    <site name="w_up" pos="0.05 0.02 0.01" euler="3 2 0"/>
    <site name="w_side" pos="0 0 0.3" euler="0 90 0"/>
    <body name="inner" pos="2 2 1">
      <site name="inside" euler="30 10 0"/>
    </body>
    {world}
    <body name="arm" pos="0 0 1.2">
      <joint name="hinge" type="hinge" axis="0 1 0" damping="0.05"/>
      <geom name="arm" type="capsule" fromto="0 0 0 0.5 0 0" size="0.03" mass="0.5"/>
      <geom name="arm_end" type="sphere" size="0.06" pos="0.6 0 0" mass="0.2"/>
      <site name="arm_down" pos="0.6 0 -0.07" euler="180 0 0"/>
      <site name="arm_tilt" pos="0.4 0 -0.04" euler="160 25 0"/>
      <site name="arm_self" pos="0.1 0 0" euler="0 90 0"/>
      <site name="arm_sky" pos="0.3 0 0.04"/>
    </body>
    <body name="sled" pos="0 0 0.9">
      <joint name="slide" type="slide" axis="1 0 0" damping="0.2"/>
      <geom name="sled" type="box" size="0.08 0.08 0.03" pos="0 0 -0.05" mass="1"/>
      <site name="sled_c" euler="0 0 0" pos="0 0 0.01"/>
      <site name="sled_down" pos="0.05 0.03 -0.09" euler="180 0 0"/>
      <site name="sled_fwd" pos="0.09 0 -0.05" euler="0 120 0"/>
      {sled}
    </body>
  </worldbody>
  <actuator>
    <motor name="m_hinge" joint="hinge" gear="0.5"/>
    <motor name="m_slide" joint="slide" gear="2"/>
  </actuator>
  <sensor>
    <jointpos joint="hinge"/>
    <jointvel joint="slide"/>
    <framepos objtype="site" objname="arm_down"/>
  </sensor>
</mujoco>"""

MESH_ASSETS = """<mesh name="tet" vertex="0 0 0  0.4 0 0  0 0.4 0  0 0 0.4" face="0 2 1  0 1 3  0 3 2  1 2 3"/>
    <mesh name="oct" vertex="0.25 0 0  -0.25 0 0  0 0.25 0  0 -0.25 0  0 0 0.3  0 0 -0.3"/>"""
MESH_WORLD = """<geom name="m_tet" type="mesh" mesh="tet" pos="0.45 -0.1 0.15" euler="0 0 20"/>
    <geom name="m_oct" type="mesh" mesh="oct" pos="-0.4 0.05 0.35" euler="10 0 0"/>
    <body name="m_body" pos="0.2 0.4 0.3"><freejoint/><geom name="m_free" type="mesh" mesh="oct" mass="0.3"/></body>"""

# rangefinder rows: (site, cutoff, nsample, delay, interval period, position among the sensors or None to append)
PRIMITIVE_ROWS = (
  ("arm_down", 0.0, 0, 0.0, 0.0, None), ("arm_tilt", 0.0, 0, 0.0, 0.0, 1), ("arm_self", 0.0, 0, 0.0, 0.0, None),
  ("arm_sky", 0.0, 0, 0.0, 0.0, None), ("arm_sky", 0.5, 0, 0.0, 0.0, None),  # a miss, and a miss under a cutoff: -1 either way
  ("sled_c", 0.0, 0, 0.0, 0.0, 0), ("sled_down", 0.0, 0, 0.0, 0.0, None), ("sled_fwd", 0.0, 0, 0.0, 0.0, None),
  ("sled_down", 5.0, 0, 0.0, 0.0, None), ("sled_down", 0.3, 0, 0.0, 0.0, None),  # cutoff above and below the hit distance
  ("w_up", 0.0, 0, 0.0, 0.0, 3), ("w_side", 0.0, 0, 0.0, 0.0, None), ("inside", 0.0, 0, 0.0, 0.0, None),
)
DELAY_ROWS = PRIMITIVE_ROWS[:2] + (
  ("arm_down", 0.0, 3, 0.004, 0.0, None), ("sled_down", 0.0, 3, 0.002, 0.0, 2), ("arm_tilt", 0.0, 2, 0.0, 0.004, None), ("sled_down", 0.3, 3, 0.006, 0.0, None),
)
MESH_ROWS = (
  ("arm_down", 0.0, 0, 0.0, 0.0, None), ("arm_tilt", 0.0, 0, 0.0, 0.0, None), ("sled_down", 0.0, 0, 0.0, 0.0, 0), ("w_up", 0.0, 0, 0.0, 0.0, None),
  ("sled_fwd", 0.0, 0, 0.0, 0.0, None),
) + tuple((f"g{i}_{j}", 0.0, 0, 0.0, 0.0, None) for i in range(3) for j in range(3))
NGRID = (15, 14)  # the `many` scene: a grid of downward sites on the sled


def _grid(nx, ny, spread=0.7):
  out = []
  for i in range(nx):
    for j in range(ny):
      x, y = spread * (i / max(nx - 1, 1) - 0.5), spread * (j / max(ny - 1, 1) - 0.5)
      out.append(f'<site name="g{i}_{j}" pos="{x:.4f} {y:.4f} -0.09" euler="{180 + 4 * (i - nx // 2)} {3 * (j - ny // 2)} 0"/>')
  return "\n      ".join(out)


def xml(integrator="Euler", mesh=False, grid=(3, 3)):
  return XML.format(integrator=integrator, assets=MESH_ASSETS if mesh else "", world=MESH_WORLD if mesh else "", sled=_grid(*grid))


def add_rangefinders(m, rows):
  """Adds rangefinders (site name, cutoff, nsample, delay, interval period, position or None) to a compiled model's sensor arrays, as MuJoCo's
  compiler lays them out: type 7 on a site, one POSITIVE output at the position stage.  A row with a position is inserted before the sensor
  at that index, and the sensordata addresses of the sensors after it move up by one."""
  from mujoco_warp_b200._src import constants as C
  from mujoco_warp_b200._src import mjcf

  for site, cutoff, nsample, delay, period, at in rows:
    ns = int(m.nsensor)
    at = ns if at is None else int(at)
    adr = int(np.asarray(m.sensor_adr)[at]) if at < ns else int(m.nsensordata)
    ins = lambda a, v: np.insert(np.asarray(a), at, v, axis=0)
    row = dict(type=C.SENS_RANGEFINDER, objtype=C.OBJ_SITE, objid=list(m.names.site).index(site), reftype=C.OBJ_UNKNOWN, refid=-1, dim=1, datatype=1, needstage=1)
    for k, v in row.items():
      setattr(m, "sensor_" + k, ins(getattr(m, "sensor_" + k), v).astype(np.int32))
    sadr = np.asarray(m.sensor_adr).copy()
    sadr[at:] += 1
    m.sensor_adr = np.insert(sadr, at, adr).astype(np.int32)
    m.sensor_intprm = ins(np.asarray(m.sensor_intprm).reshape(-1, 3), np.zeros(3, dtype=np.int32)).astype(np.int32)
    m.sensor_cutoff, m.sensor_noise = ins(m.sensor_cutoff, cutoff), ins(m.sensor_noise, 0.0)
    m.sensor_history = ins(np.asarray(m.sensor_history).reshape(-1, 2), [nsample, 0]).astype(np.int32)
    m.sensor_delay = ins(m.sensor_delay, delay)
    m.sensor_interval = ins(np.asarray(m.sensor_interval).reshape(-1, 2), [period, 0.0])
    m.names.sensor = list(m.names.sensor)[:at] + [f"rangefinder{ns}"] + list(m.names.sensor)[at:]
    m.nsensor = ns + 1
    m.nsensordata = int(m.nsensordata) + 1
  mjcf.set_history_layout(m)
  return m


def _load(integrator="Euler", rows=PRIMITIVE_ROWS, mesh=False, grid=(3, 3)):
  from mujoco_warp_b200._src import mjcf

  return add_rangefinders(mjcf.load_string(xml(integrator, mesh, grid)), rows)


def _many_rows():
  return tuple((f"g{i}_{j}", 0.0, 0, 0.0, 0.0, None) for i in range(NGRID[0]) for j in range(NGRID[1]))


INTEGRATORS = {"implicitfast": "implicitfast", "implicit": "implicit", "rk4": "RK4"}
# name: (model source, steps, per-world fields)
SCENES = {
  "primitives": (lambda: _load("Euler"), 6, False),
  "mesh": (lambda: _load("Euler", MESH_ROWS, mesh=True), 4, False),
  "delay": (lambda: _load("Euler", DELAY_ROWS), 6, False),
  "batched": (lambda: _load("Euler"), 4, True),
  **{k: ((lambda i: lambda: _load(i))(v), 4, False) for k, v in INTEGRATORS.items()},
  "many": (lambda: _load("Euler", _many_rows(), grid=NGRID), 2, False),
}


def load(name):
  return SCENES[name][0]()


def batched(mjm, nworld=NWORLD):
  """Per-world geom_size (nworld, ngeom, 3) and geom_rgba (nworld, ngeom, 4): sizes scaled per world, and the static sphere / box and the
  sled's box transparent in some worlds only."""
  k = np.arange(nworld, dtype=np.float64)
  size = np.asarray(mjm.geom_size, dtype=np.float64)[None] * (1.0 + 0.15 * k[:, None, None])
  rgba = np.tile(np.asarray(mjm.geom_rgba, dtype=np.float64)[None], (nworld, 1, 1))
  names = list(mjm.names.geom)
  rgba[1, names.index("s_sphere"), 3] = 0.0
  rgba[nworld - 1, names.index("s_box"), 3] = 0.0
  rgba[0, names.index("floor"), 3] = 0.0
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(size), f32(rgba)


def seeded(mjm, nsteps, nworld=NWORLD, seed=5):
  """Per-world qpos / qvel and a per-world, per-step ctrl (nsteps, nworld, nu), fp32-representable."""
  from tests import util

  qpos, qvel, _, _ = util.seeded_state(mjm, nworld, key=None, seed=seed, qpos_noise=0.6, qvel_noise=1.0, exact_world0=False)
  rng = np.random.default_rng(seed)
  ctrl = rng.uniform(-1.0, 1.0, (nsteps, nworld, int(mjm.nu)))
  f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
  return f32(qpos), f32(qvel), f32(ctrl)
