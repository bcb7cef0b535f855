"""MJCF scenes with <contact> sensors, shared by the contact-sensor tests, tools/make_contact_sensor_goldens.py and
tools/contact_sensor_bench.py.

Bodies on a plane: a box resting on its face (four contacts), a sphere and a capsule sliding, and a cart whose child wheel also touches
the floor (so that a subtree has contacts on two bodies).  The sensors between them cover every data keyword alone and all together, each
reduction at num 1, 3 and more than the matches, and matching with no object, geom1, body1, subtree1, geom2 only and both sides in both
orders; `site_xml` adds a site volume of each primitive type.  `humanoid` adds foot sensors to the benchmark humanoid."""

import numpy as np

DATA = ("found", "force", "torque", "dist", "pos", "normal", "tangent")
ALL = " ".join(DATA)


def _bodies(condim=(3, 3, 3, 3)):
  cb, cs, cc, cw = condim
  return f"""
    <geom name="floor" type="plane" size="3 3 .1"/>
    <body name="box" pos="0 0 .098"><freejoint/><geom name="box" type="box" size=".1 .1 .1" condim="{cb}"/></body>
    <body name="ball" pos=".5 0 .099"><freejoint/><geom name="ball" type="sphere" size=".1" condim="{cs}"/></body>
    <body name="capsule" pos="-.5 0 .099" euler="0 90 0"><freejoint/><geom name="capsule" type="capsule" size=".1 .2" condim="{cc}"/></body>
    <body name="cart" pos="0 .6 .149">
      <freejoint/><geom name="cart" type="box" size=".2 .1 .05" pos="0 0 0" condim="3"/>
      <body name="wheel" pos=".3 0 -.05"><joint name="wheel" type="hinge" axis="0 1 0"/><geom name="wheel" type="sphere" size=".1" condim="{cw}"/></body>
    </body>"""


def _contact(name, data=ALL, reduce="none", num=1, **sides):
  attrs = " ".join(f'{k}="{v}"' for k, v in sides.items())
  return f'<contact name="{name}" {attrs} data="{data}" reduce="{reduce}" num="{num}"/>'


def _sensors_main():
  s = [_contact(f"alone_{k}", data=k, num=3) for k in DATA]  # every keyword alone, all contacts
  for reduce in ("none", "mindist", "maxforce", "netforce"):
    for num in (1, 3, 7):
      s.append(_contact(f"box_{reduce}_{num}", reduce=reduce, num=num, body1="box"))
      s.append(_contact(f"all_{reduce}_{num}", data="found force dist", reduce=reduce, num=num))
  s += [
    _contact("geom1", geom1="ball", num=2),
    _contact("subtree1", subtree1="cart", reduce="maxforce", num=4),
    _contact("subtree1_net", subtree1="cart", reduce="netforce"),
    _contact("body1_child", body1="wheel", num=2),
    _contact("geom2_only", geom2="capsule", num=2),
    _contact("floor_box", geom1="floor", geom2="box", reduce="mindist", num=4),
    _contact("box_floor", geom1="box", geom2="floor", reduce="mindist", num=4),
    _contact("floor_subtree", body1="world", subtree2="cart", num=3),
    _contact("subtree_floor", subtree1="cart", body2="world", num=3),
    _contact("box_floor_net", body1="box", geom2="floor", reduce="netforce"),
    _contact("nomatch", geom1="ball", geom2="box"),
  ]
  return "\n    ".join(s)


def main_xml(cone="pyramidal", condim=(3, 3, 3, 3), extra_sensors="", custom=""):
  return f"""
<mujoco model="contact_sensor">
  <option timestep="0.004" cone="{cone}"/>
  {custom}
  <worldbody>{_bodies(condim)}
  </worldbody>
  <sensor>
    {_sensors_main()}
    {extra_sensors}
  </sensor>
</mujoco>"""


def site_xml():
  """a site volume of each type around a contact region, in the world body and on a moving body"""
  sites = """
    <site name="s_sphere" type="sphere" size=".25" pos="0 0 0"/>
    <site name="s_capsule" type="capsule" size=".15 .3" pos="-.5 0 0" euler="0 90 0"/>
    <site name="s_ellipsoid" type="ellipsoid" size=".3 .12 .1" pos=".5 0 0"/>
    <site name="s_cylinder" type="cylinder" size=".12 .05" pos="0 0 0"/>
    <site name="s_box" type="box" size=".35 .12 .05" pos=".15 .6 0"/>"""
  sensors = "\n    ".join(_contact(f"site_{t}", site=f"s_{t}", num=5, reduce=r) for t, r in
                          (("sphere", "none"), ("capsule", "mindist"), ("ellipsoid", "none"), ("cylinder", "maxforce"), ("box", "netforce")))
  sensors += "\n    " + _contact("site_box_floor", site="s_box", geom2="floor", num=3)
  return f"""
<mujoco model="contact_sensor_sites">
  <option timestep="0.004"/>
  <worldbody>{_bodies()}{sites}
  </worldbody>
  <sensor>
    {sensors}
  </sensor>
</mujoco>"""


def overflow_xml(maxmatch=3, netforce=False):
  """a match capacity below the scene's contact count.  Without `netforce` the sensors keep num <= maxmatch and no netforce: the
  reference reads past its match buffer otherwise, so only those have fixtures."""
  s = [_contact("all_none_1"), _contact("all_none_3", num=3), _contact("all_mindist_2", reduce="mindist", num=2),
       _contact("all_maxforce_3", reduce="maxforce", num=3), _contact("box_none_3", body1="box", num=3)]
  if netforce:
    s += [_contact("all_netforce", reduce="netforce", num=2), _contact("all_none_6", num=6), _contact("all_mindist_6", reduce="mindist", num=6)]
  return f"""
<mujoco model="contact_sensor_overflow">
  <option timestep="0.004"/>
  <custom><numeric name="contact_sensor_maxmatch" data="{maxmatch}"/></custom>
  <worldbody>{_bodies()}
  </worldbody>
  <sensor>
    {chr(10).join(s)}
  </sensor>
</mujoco>"""


def delay_xml():
  """a delayed contact sensor next to its undelayed twin"""
  extra = ('<contact name="box_delayed" body1="box" data="found force" num="4" nsample="3" delay="0.004"/>\n    '
           '<contact name="box_fresh" body1="box" data="found force" num="4"/>')
  return main_xml(extra_sensors=extra)


# name -> (xml, make_data njmax) of the scenes with reference fixtures
SCENES = {
  "pyramidal": (main_xml(), 256),
  "pyramidal_condim": (main_xml(condim=(6, 1, 3, 6)), 256),
  "elliptic_condim": (main_xml(cone="elliptic", condim=(6, 1, 3, 6)), 256),
  "sites": (site_xml(), 256),
  "overflow": (overflow_xml(), 256),
  "njmax": (main_xml(), 20),  # cuts the contact rows of the later contacts
  "delay": (delay_xml(), 256),
}

# the benchmark humanoid's foot sensors: subtree1 on each foot, found + force, netforce and maxforce
HUMANOID_FEET = (("foot_right", "netforce"), ("foot_left", "netforce"), ("foot_right", "maxforce"), ("foot_left", "maxforce"))


def humanoid(feet=HUMANOID_FEET, num=1):
  """the benchmark humanoid (no sensors of its own) with contact sensors appended: subtree1 on the named bodies, data found + force"""
  from mujoco_warp_b200._src import constants as C
  from mujoco_warp_b200._src import mjcf
  from mujoco_warp_b200.scenes import HUMANOID

  m = mjcf.load_any(HUMANOID)
  assert m.nsensor == 0
  n = len(feet)
  size = mjcf.contact_slot_size(3)
  m.nsensor = n
  m.names.sensor = [f"{b}_{r}" for b, r in feet]
  m.sensor_type = np.full(n, C.SENS_CONTACT, dtype=np.int32)
  m.sensor_objtype = np.full(n, C.OBJ_XBODY, dtype=np.int32)
  m.sensor_objid = np.array([m.names.body.index(b) for b, _ in feet], dtype=np.int32)
  m.sensor_reftype = np.zeros(n, dtype=np.int32)
  m.sensor_refid = -np.ones(n, dtype=np.int32)
  m.sensor_intprm = np.array([(3, mjcf.CONTACT_REDUCE.index(r), num) for _, r in feet], dtype=np.int32)
  m.sensor_dim = np.full(n, num * size, dtype=np.int32)
  m.sensor_datatype = np.zeros(n, dtype=np.int32)
  m.sensor_needstage = np.full(n, 3, dtype=np.int32)
  m.sensor_cutoff = np.zeros(n)
  m.sensor_noise = np.zeros(n)
  m.sensor_adr = (np.arange(n) * num * size).astype(np.int32)
  m.nsensordata = int(n * num * size)
  m.sensor_unsupported = []
  return m
