"""MJCF scenes with fluid forces (density, viscosity, wind), shared by the fluid tests and tools/make_fluid_goldens.py."""


def chain_xml(integrator="Euler", density=1000.0, viscosity=0.01, wind="0.3 -0.2 0.1"):
  """A free-floating chain of capsules and a box linked by hinges and a ball joint (a swimmer): the inertia-box model on every body."""
  return f"""
<mujoco model="fluid_chain">
  <option timestep="0.002" integrator="{integrator}" density="{density}" viscosity="{viscosity}" wind="{wind}" gravity="0 0 -2"/>
  <default><geom contype="0" conaffinity="0" density="900"/><joint damping="0.002"/></default>
  <worldbody>
    <body name="head" pos="0 0 1">
      <freejoint/>
      <geom type="capsule" fromto="0 0 0 0.12 0 0" size="0.03"/>
      <body name="seg1" pos="0.12 0 0">
        <joint name="h1" type="hinge" axis="0 0 1" range="-90 90"/>
        <geom type="capsule" fromto="0 0 0 0.1 0 0" size="0.025"/>
        <body name="seg2" pos="0.1 0 0">
          <joint name="h2" type="hinge" axis="0 1 0"/>
          <geom type="box" size="0.05 0.02 0.01" pos="0.05 0 0"/>
          <body name="tail" pos="0.1 0 0">
            <joint name="b3" type="ball"/>
            <geom type="ellipsoid" size="0.06 0.015 0.03" pos="0.06 0 0"/>
          </body>
        </body>
      </body>
    </body>
  </worldbody>
  <actuator><motor joint="h1" gear="0.05"/><motor joint="h2" gear="0.05"/></actuator>
</mujoco>"""


def ellipsoid_xml(integrator="Euler"):
  """The ellipsoid model on every geom type: sphere, capsule, cylinder, box, ellipsoid and mesh, non-default coefficients, a body that
  mixes ellipsoid and fluidshape="none" geoms, and a massless body."""
  return f"""
<mujoco model="fluid_ellipsoid">
  <option timestep="0.002" integrator="{integrator}" density="1.2" viscosity="0.00002" wind="0.5 0 -0.3" gravity="0 0 -9.81"/>
  <default>
    <geom contype="0" conaffinity="0" fluidshape="ellipsoid" fluidcoef="0.4 0.3 1.2 0.8 1.1"/>
    <default class="plain"><geom fluidshape="none"/></default>
  </default>
  <asset>
    <mesh name="tet" vertex="0 0 0  0.08 0 0  0 0.06 0  0 0 0.05  0.04 0.04 0.04"/>
  </asset>
  <worldbody>
    <body name="ball" pos="0 0 1">
      <freejoint/>
      <geom type="sphere" size="0.05"/>
      <body name="arm" pos="0 0 0.05">
        <joint type="hinge" axis="1 0 0"/>
        <geom type="capsule" fromto="0 0 0 0 0 0.1" size="0.02" fluidcoef="0.5 0.2 1.5 1.3 0.7"/>
        <body name="fin" pos="0 0 0.12">
          <joint type="hinge" axis="0 1 0"/>
          <geom type="cylinder" size="0.03 0.01"/>
          <geom class="plain" type="box" size="0.01 0.04 0.005" pos="0 0 0.02"/>
          <geom type="box" size="0.04 0.02 0.006" pos="0.02 0 0.03"/>
          <body name="tag" pos="0 0.05 0">
            <geom type="sphere" size="0.01" density="0" mass="0"/>
          </body>
        </body>
      </body>
    </body>
    <body name="egg" pos="0.5 0 1">
      <freejoint/>
      <geom type="ellipsoid" size="0.06 0.03 0.02"/>
      <body name="rock" pos="0 0 0.08">
        <joint type="ball"/>
        <geom type="mesh" mesh="tet" density="2000"/>
      </body>
    </body>
  </worldbody>
</mujoco>"""


def sphere_xml(radius=0.05, density_geom=2000.0, viscosity=2.0, integrator="Euler"):
  """One free sphere falling in a viscous fluid (inertia-box model)."""
  return f"""
<mujoco model="fluid_sphere">
  <option timestep="0.002" integrator="{integrator}" viscosity="{viscosity}" gravity="0 0 -9.81"/>
  <worldbody>
    <body name="ball" pos="0 0 0">
      <freejoint/>
      <geom type="sphere" size="{radius}" density="{density_geom}" contype="0" conaffinity="0"/>
    </body>
  </worldbody>
</mujoco>"""


# fixture scene -> (xml, nworld)
SCENES = {
  "chain": (chain_xml(), 3),
  "ellipsoid": (ellipsoid_xml(), 3),
  "ellipsoid_implicitfast": (ellipsoid_xml("implicitfast"), 3),
  "chain_rk4": (chain_xml("RK4"), 3),
  "density_only": (chain_xml(density=1000.0, viscosity=0.0, wind="0 0 0"), 3),
  "viscosity_only": (chain_xml(density=0.0, viscosity=0.5, wind="0 0 0"), 3),
  "wind_only": (chain_xml(density=0.0, viscosity=0.0, wind="1 0 0"), 3),
}
