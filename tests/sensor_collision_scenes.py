"""MJCF scenes with distance / normal / fromto sensors, shared by the collision-sensor tests and tools/sensor_collision_bench.py."""

SENSORS = ("distance", "normal", "fromto")


def _sensors(pairs):
  """Every sensor tag for every (side1, side2, cutoff); a side is ("geom" | "body", name)."""
  return "\n".join(f'<{tag} {k1}1="{n1}" {k2}2="{n2}" cutoff="{c}"/>' for tag in SENSORS for (k1, n1), (k2, n2), c in pairs)


def pair_xml(type0="sphere", type1="sphere", type2="box", type3="capsule", contype=0, nativeccd=True):
  """Three free bodies as in the reference's sensor tests: obj0, obj1 one geom each, objobj two geoms; sensors geom-geom, geom-body and
  body-body, both orders, cutoffs 0 and 10."""
  flag = "" if nativeccd else '<option><flag nativeccd="disable"/></option>'
  pairs = []
  for a, b in ((("geom", "obj0"), ("geom", "obj1")), (("geom", "obj0"), ("body", "objobj")), (("body", "obj1"), ("body", "objobj"))):
    for c in (0, 10):
      pairs += [(a, b, c), (b, a, c)]
  return f"""
<mujoco model="sensor_collision_pair">
  {flag}
  <default><geom contype="{contype}" conaffinity="{contype}"/></default>
  <worldbody>
    <body name="obj0"><freejoint/><geom name="obj0" type="{type0}" size=".1 .1 .1" euler="1 2 3"/></body>
    <body name="obj1" pos="0 0 1"><freejoint/><geom name="obj1" type="{type1}" size=".1 .1 .1" euler="-1 2 -1"/></body>
    <body name="objobj" pos="0 0 -1">
      <freejoint/>
      <geom name="objobj0" pos=".01 0 0.005" type="{type2}" size=".09 .09 .09" euler="2 1 3"/>
      <geom name="objobj1" pos="-.01 0 -0.0025" type="{type3}" size=".11 .11 .11" euler="3 1 2"/>
    </body>
  </worldbody>
  <sensor>
    {_sensors(pairs)}
  </sensor>
</mujoco>"""


def plane_xml(type_="sphere"):
  """A tilted plane and one free geom, as the reference's plane sensor test."""
  pairs = [(("geom", "plane"), ("geom", "obj"), 0), (("geom", "plane"), ("geom", "obj"), 10), (("geom", "obj"), ("geom", "plane"), 0),
           (("geom", "obj"), ("geom", "plane"), 10), (("geom", "plane"), ("body", "obj"), 10)]
  return f"""
<mujoco model="sensor_collision_plane">
  <worldbody>
    <geom name="plane" type="plane" size="10 10 .01" euler="2 2 2" contype="0" conaffinity="0"/>
    <body name="obj" pos="0 0 1"><freejoint/><geom name="obj" type="{type_}" size=".1 .1 .1" euler="1 2 3" contype="0" conaffinity="0"/></body>
  </worldbody>
  <sensor>
    {_sensors(pairs)}
  </sensor>
</mujoco>"""


def spheres_xml(r1=0.1, r2=0.15, contact=False, sensors=True, cutoff=10):
  """Two free spheres over a ground plane: the analytic cases (sphere-sphere, sphere-plane), optionally colliding with each other."""
  c = 1 if contact else 0
  sens = f"""<sensor>
    <distance geom1="a" geom2="b" cutoff="{cutoff}"/><normal geom1="a" geom2="b" cutoff="{cutoff}"/><fromto geom1="a" geom2="b" cutoff="{cutoff}"/>
    <distance geom1="b" geom2="a" cutoff="{cutoff}"/><normal geom1="b" geom2="a" cutoff="{cutoff}"/><fromto geom1="b" geom2="a" cutoff="{cutoff}"/>
    <distance geom1="floor" geom2="a" cutoff="{cutoff}"/><fromto geom1="floor" geom2="a" cutoff="{cutoff}"/><normal geom1="a" geom2="floor" cutoff="{cutoff}"/>
  </sensor>""" if sensors else ""
  return f"""
<mujoco model="sensor_collision_spheres">
  <option timestep="0.002"/>
  <worldbody>
    <geom name="floor" type="plane" size="5 5 .1" contype="1" conaffinity="1"/>
    <body name="a" pos="0 0 0.5"><freejoint/><geom name="a" type="sphere" size="{r1}" contype="{c}" conaffinity="1"/></body>
    <body name="b" pos="0.3 0.1 0.6"><freejoint/><geom name="b" type="sphere" size="{r2}" contype="{c}" conaffinity="1"/></body>
  </worldbody>
  {sens}
</mujoco>"""


def mesh_xml():
  """The three-body scene with a tetrahedron-like mesh as objobj0 (mesh-box, mesh-capsule, plane-free GJK / EPA pairs)."""
  return pair_xml("box", "capsule", "mesh", "cylinder").replace(
    "<worldbody>", '<asset><mesh name="m" vertex="0 0 0  .1 0 0  0 .1 0  0 0 .1  .05 .05 .05"/></asset><worldbody>').replace(
    'type="mesh" size=".09 .09 .09"', 'type="mesh" mesh="m"')


def overlap_xml():
  """Overlapping pairs (negative distances): ellipsoid-cylinder and box-box through GJK / EPA, capsule-capsule through its primitive."""
  pairs = [(("geom", "e"), ("geom", "c"), 10), (("geom", "c"), ("geom", "e"), 10), (("geom", "b1"), ("geom", "b2"), 10),
           (("geom", "k1"), ("geom", "k2"), 10), (("geom", "k2"), ("geom", "k1"), 1)]
  return f"""
<mujoco model="sensor_collision_overlap">
  <default><geom contype="0" conaffinity="0"/></default>
  <worldbody>
    <body name="e" pos="0 0 0"><freejoint/><geom name="e" type="ellipsoid" size=".12 .08 .1" euler="0.3 0.2 0.1"/></body>
    <body name="c" pos="0.1 0.02 0.05"><freejoint/><geom name="c" type="cylinder" size=".08 .1" euler="0.5 -0.2 0"/></body>
    <body name="b1" pos="2 0 0"><freejoint/><geom name="b1" type="box" size=".1 .1 .1" euler="0.1 0.2 0.3"/></body>
    <body name="b2" pos="2.12 0.03 0.05"><freejoint/><geom name="b2" type="box" size=".08 .09 .1" euler="-0.2 0.4 0.1"/></body>
    <body name="k1" pos="-2 0 0"><freejoint/><geom name="k1" type="capsule" size=".05 .2" euler="0 1.2 0"/></body>
    <body name="k2" pos="-2 0.03 0.06"><freejoint/><geom name="k2" type="capsule" size=".05 .15" euler="1.1 0 0.3" margin="0.05"/></body>
  </worldbody>
  <sensor>
    {_sensors(pairs)}
  </sensor>
</mujoco>"""


def contact_xml():
  """A sensor pair that is also a contact pair (two resting spheres and a box on the floor), and a parent-child pair that the
  contact filter excludes (a hinged capsule and its parent box)."""
  pairs = [(("geom", "a"), ("geom", "b"), 10), (("geom", "floor"), ("body", "b"), 10), (("geom", "arm"), ("geom", "base"), 10),
           (("body", "base"), ("body", "armb"), 0.05)]
  return f"""
<mujoco model="sensor_collision_contact">
  <option timestep="0.002"/>
  <worldbody>
    <geom name="floor" type="plane" size="5 5 .1"/>
    <body name="a" pos="0 0 0.1"><freejoint/><geom name="a" type="sphere" size=".1"/></body>
    <body name="b" pos="0.19 0 0.1"><freejoint/><geom name="b" type="sphere" size=".1"/><geom name="bb" type="box" size=".05 .05 .05" pos="0 0 .12"/></body>
    <body name="base" pos="1 0 0.3">
      <freejoint/>
      <geom name="base" type="box" size=".1 .1 .1"/>
      <body name="armb" pos="0 0 .1"><joint type="hinge" axis="1 0 0"/><geom name="arm" type="capsule" fromto="0 0 0 0 .2 .1" size=".04"/></body>
    </body>
  </worldbody>
  <sensor>
    {_sensors(pairs)}
  </sensor>
</mujoco>"""


def _fixture_scenes():
  out = {}
  for types in (("box", "box", "box", "box"), ("sphere", "capsule", "ellipsoid", "cylinder"), ("capsule", "box", "cylinder", "sphere"),
                ("capsule", "cylinder", "box", "ellipsoid"), ("cylinder", "box", "ellipsoid", "capsule")):
    out["pair_" + "_".join(types)] = pair_xml(*types)
  for t in ("sphere", "capsule", "ellipsoid", "cylinder", "box"):
    out["plane_" + t] = plane_xml(t)
  out["mesh"], out["overlap"], out["contact"] = mesh_xml(), overlap_xml(), contact_xml()
  return out


# the reference-generated fixtures tests/golden/sensor_collision_<name>.npz (tools/make_sensor_collision_goldens.py), 3 worlds each
SCENES = _fixture_scenes()
