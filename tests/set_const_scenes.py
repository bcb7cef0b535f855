"""Scenes for set_const (tests/test_set_const_host.py, tests/test_gpu_set_const.py, tools/make_set_const_goldens.py).

Each scene is an MJCF string and the per-world inputs of its worlds: the fields a user randomises per world before calling set_const.
Every output field is batched to NWORLD as well, so entry w of each output is world w's result.  `unbatched` runs the same call
with every field shared by all worlds (world 0's result lands in the single entry).
"""
import numpy as np

NWORLD = 3

CHAIN = """
<mujoco model="chain">
  <worldbody>
    <geom type="plane" size="0 0 .05"/>
    <body name="l0" pos="0 0 1">
      <joint name="j0" type="hinge" axis="0 1 0"/>
      <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03"/>
      <body name="l1" pos="0.3 0 0">
        <joint name="j1" type="hinge" axis="0 1 0" armature="0.01"/>
        <geom type="capsule" fromto="0 0 0 0.25 0 0" size="0.025"/>
        <body name="l2" pos="0.25 0 0">
          <joint name="j2" type="hinge" axis="1 0 0"/>
          <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.02"/>
        </body>
      </body>
    </body>
  </worldbody>
  <actuator>
    <motor joint="j0" gear="2"/> <motor joint="j1" gear="1"/> <motor joint="j2" gear="0.5"/>
  </actuator>
</mujoco>"""

MIXED = """
<mujoco model="mixed">
  <worldbody>
    <geom type="plane" size="0 0 .05"/>
    <body name="torso" pos="0 0 1">
      <freejoint/>
      <geom type="box" size="0.1 0.08 0.05"/>
      <body name="arm" pos="0.1 0 0">
        <joint name="shoulder" type="ball"/>
        <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.03"/>
        <body name="forearm" pos="0.2 0 0">
          <joint name="elbow" type="hinge" axis="0 0 1"/>
          <geom type="capsule" fromto="0 0 0 0.15 0 0" size="0.025"/>
        </body>
      </body>
    </body>
    <body name="pend" pos="1 0 1">
      <joint name="swing" type="hinge" axis="0 1 0"/>
      <geom type="sphere" size="0.05" pos="0 0 -0.3"/>
    </body>
  </worldbody>
  <actuator>
    <motor joint="elbow" gear="3"/> <motor joint="swing"/>
  </actuator>
</mujoco>"""

STATIC = """
<mujoco model="static">
  <worldbody>
    <geom type="plane" size="0 0 .05"/>
    <body name="wall" pos="0.5 0 0.5"><geom type="box" size="0.05 0.5 0.5"/></body>
    <body name="slider" pos="0 0 0.3">
      <joint name="sx" type="slide" axis="1 0 0"/>
      <geom type="box" size="0.05 0.05 0.05"/>
      <body name="rider" pos="0 0 0.1"><geom type="sphere" size="0.03"/></body>
    </body>
    <body name="xy" pos="0 1 0.3">
      <joint name="x" type="slide" axis="1 0 0"/> <joint name="y" type="slide" axis="0 1 0"/>
      <geom type="sphere" size="0.05"/>
    </body>
    <body name="arm" pos="-1 0 1">
      <joint name="h" type="hinge" axis="0 0 1"/>
      <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03"/>
    </body>
  </worldbody>
  <actuator><motor joint="sx"/></actuator>
</mujoco>"""

EQUALITY = """
<mujoco model="eq">
  <worldbody>
    <body name="a" pos="0 0 1">
      <joint name="ha" type="hinge" axis="0 1 0"/>
      <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.02"/>
      <body name="a2" pos="0.3 0 0">
        <joint name="ha2" type="hinge" axis="0 1 0"/>
        <geom type="capsule" fromto="0 0 0 0 0 -0.3" size="0.02"/>
      </body>
    </body>
    <body name="b" pos="0.3 0 0.6">
      <joint name="hb" type="hinge" axis="0 1 0"/>
      <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.02"/>
    </body>
    <body name="f1" pos="0.6 0.5 0.5"><freejoint/><geom type="sphere" size="0.05"/></body>
    <body name="f2" pos="0.8 0.5 0.6" euler="10 20 30"><freejoint/><geom type="box" size="0.04 0.04 0.04"/></body>
    <body name="f3" pos="0.8 -0.5 0.6"><freejoint/><geom type="box" size="0.04 0.04 0.04"/></body>
  </worldbody>
  <equality>
    <connect body1="a2" body2="b" anchor="0 0 -0.3"/>
    <weld body1="f1" body2="f2" anchor="0.1 0 0"/>
    <weld body1="f2" body2="f3"/>
    <connect body1="f3" anchor="0 0.1 0"/>
  </equality>
</mujoco>"""

CAMLIGHT = """
<mujoco model="camlight">
  <worldbody>
    <light name="lfix" pos="0 0 3" dir="0 0 -1"/>
    <camera name="cfix" pos="2 0 1" euler="0 80 0"/>
    <body name="base" pos="0 0 1">
      <joint name="bx" type="slide" axis="1 0 0"/>
      <joint name="bz" type="hinge" axis="0 0 1"/>
      <geom type="box" size="0.1 0.1 0.1"/>
      <camera name="ctrack" mode="track" pos="0.5 0 0.2"/>
      <camera name="ctrackcom" mode="trackcom" pos="0 0.5 0.3"/>
      <light name="ltrack" mode="track" pos="0 0 0.5" dir="0 0.3 -1"/>
      <light name="ltrackcom" mode="trackcom" pos="0.2 0 0.5" dir="0 0 -1"/>
      <light name="laim" mode="targetbody" target="tip" pos="-0.3 0.2 0.6"/>
      <light name="laimcom" mode="targetbodycom" target="tip" pos="0.3 -0.2 0.7"/>
      <body name="tip" pos="0.3 0 0">
        <joint name="ty" type="hinge" axis="0 1 0"/>
        <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03"/>
        <camera name="ctarget" mode="targetbody" target="base" pos="0.2 0.3 0.4"/>
        <camera name="ctargetcom" mode="targetbodycom" target="base" pos="-0.2 0.3 0.4"/>
      </body>
    </body>
  </worldbody>
</mujoco>"""

TENDON = """
<mujoco model="tendon">
  <worldbody>
    <body name="a0" pos="0 0 0.6">
      <joint name="a0" type="hinge" axis="0 1 0"/>
      <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.03"/>
      <body name="a1" pos="0.2 0 0">
        <joint name="a1" type="hinge" axis="0 1 0"/>
        <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.025"/>
      </body>
    </body>
    <body name="s" pos="-0.4 0 0.3">
      <joint name="pz" type="slide" axis="0 0 1"/>
      <geom type="box" size="0.05 0.04 0.02"/>
    </body>
  </worldbody>
  <tendon>
    <fixed name="t0" stiffness="5"><joint joint="a0" coef="0.5"/><joint joint="a1" coef="-0.5"/></fixed>
    <fixed name="t1" stiffness="2" springlength="0.1 0.2"><joint joint="a1" coef="1"/><joint joint="pz" coef="0.7"/></fixed>
    <fixed name="t2"><joint joint="pz" coef="2"/></fixed>
  </tendon>
  <actuator>
    <motor tendon="t0" gear="2"/> <motor joint="pz"/>
  </actuator>
</mujoco>"""

DAMPRATIO = """
<mujoco model="dampratio">
  <worldbody>
    <body name="a" pos="0 0 1">
      <joint name="ha" type="hinge" axis="0 1 0" armature="0.02"/>
      <geom type="capsule" fromto="0 0 0 0.3 0 0" size="0.03"/>
      <body name="b" pos="0.3 0 0">
        <joint name="hb" type="hinge" axis="0 0 1"/>
        <geom type="capsule" fromto="0 0 0 0.2 0 0" size="0.02"/>
      </body>
    </body>
    <body name="s" pos="1 0 1"><joint name="sz" type="slide" axis="0 0 1"/><geom type="sphere" size="0.1"/></body>
  </worldbody>
  <tendon><fixed name="t"><joint joint="ha" coef="1"/><joint joint="hb" coef="0.5"/></fixed></tendon>
  <actuator>
    <general name="pr" joint="ha" gainprm="20" biastype="affine" biasprm="0 -20 0.7"/>
    <general name="pr2" joint="sz" gear="2" gainprm="50" biastype="affine" biasprm="0 -50 1.2"/>
    <general name="prt" tendon="t" gainprm="10" biastype="affine" biasprm="0 -10 0.5"/>
    <position name="pkv" joint="hb" kp="10" kv="0.3"/>
    <general name="notdr" joint="hb" gainprm="5" biastype="affine" biasprm="0 -4 0.5"/>
  </actuator>
</mujoco>"""


def _scale(rng, shape, lo=0.6, hi=1.6):
  return rng.uniform(lo, hi, size=shape)


def per_world_inputs(name, mjm, nworld=NWORLD, seed=7):
  """{Model field: (nworld, ...) float64} the scene randomises per world."""
  rng = np.random.default_rng(seed)
  tile = lambda a: np.repeat(np.asarray(a, dtype=np.float64)[None], nworld, axis=0)
  out = {}
  if name == "unbatched":
    return out
  if name in ("chain", "static", "camlight", "dampratio"):
    out["body_mass"] = tile(mjm.body_mass) * _scale(rng, (nworld, mjm.nbody))
  if name == "mixed":
    out["body_ipos"] = tile(mjm.body_ipos) + rng.normal(0, 0.02, (nworld, mjm.nbody, 3))
    out["body_inertia"] = tile(mjm.body_inertia) * _scale(rng, (nworld, mjm.nbody, 3), 0.8, 1.3)
    out["dof_armature"] = tile(mjm.dof_armature) + rng.uniform(0, 0.05, (nworld, mjm.nv))
    q0 = tile(mjm.qpos0)
    q0[:, 0:3] += rng.normal(0, 0.1, (nworld, 3))
    quat = rng.normal(0, 1, (nworld, 4))
    q0[:, 3:7] = quat / np.linalg.norm(quat, axis=1, keepdims=True)
    ball = rng.normal(0, 1, (nworld, 4))
    ball[:, 0] += 3
    q0[:, 7:11] = ball / np.linalg.norm(ball, axis=1, keepdims=True)
    q0[:, 11:] += rng.normal(0, 0.4, (nworld, mjm.nq - 11))
    out["qpos0"] = q0
  if name in ("equality", "camlight", "chain"):
    q0 = tile(mjm.qpos0)
    free = [j for j in range(mjm.njnt) if mjm.jnt_type[j] == 0]
    for j in range(mjm.njnt):
      a = mjm.jnt_qposadr[j]
      if mjm.jnt_type[j] in (2, 3):
        q0[:, a] += rng.normal(0, 0.3, nworld)
    for j in free:
      a = mjm.jnt_qposadr[j]
      q0[:, a : a + 3] += rng.normal(0, 0.1, (nworld, 3))
      quat = rng.normal(0, 1, (nworld, 4))
      quat[:, 0] += 2
      q0[:, a + 3 : a + 7] = quat / np.linalg.norm(quat, axis=1, keepdims=True)
    out["qpos0"] = q0
  if name == "equality":
    ed = tile(mjm.eq_data)
    ed[:, 2, 6:10] = 0.0  # weld f2-f3: quaternion cleared -> relative pose recomputed
    ed[:, 1, 6:10] = np.array([2.0, 0.1, 0.0, 0.0]) * rng.uniform(0.5, 2.0, (nworld, 1))  # weld f1-f2: set, only normalised
    out["eq_data"] = ed
  if name == "tendon":
    ls = tile(mjm.tendon_lengthspring)
    ls[:, 0] = -1.0  # t0: resolved at qpos_spring
    ls[:, 2] = -1.0  # t2 as well
    out["tendon_lengthspring"] = ls
    qs = tile(mjm.qpos_spring) + rng.normal(0, 0.3, (nworld, mjm.nq))
    out["qpos_spring"] = qs
    out["body_mass"] = tile(mjm.body_mass) * _scale(rng, (nworld, mjm.nbody))
  if name == "dampratio":
    gp = tile(mjm.actuator_gainprm)
    bp = tile(mjm.actuator_biasprm)
    k = _scale(rng, (nworld,), 0.5, 2.0)
    gp[:, 0, 0] *= k
    bp[:, 0, 1] *= k  # still gainprm[0] == -biasprm[1]
    out["actuator_gainprm"] = gp
    out["actuator_biasprm"] = bp
  return out


SCENES = {
  "chain": CHAIN, "mixed": MIXED, "static": STATIC, "equality": EQUALITY, "camlight": CAMLIGHT, "tendon": TENDON, "dampratio": DAMPRATIO,
  "unbatched": CHAIN,
}
# derived fields written by set_const (besides stat.meaninertia)
OUTPUTS = ("body_subtreemass", "tendon_length0", "eq_data", "dof_invweight0", "body_invweight0", "tendon_invweight0", "cam_pos0", "cam_poscom0",
           "cam_mat0", "light_pos0", "light_poscom0", "light_dir0", "actuator_acc0", "actuator_biasprm", "tendon_lengthspring")
