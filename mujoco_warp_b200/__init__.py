"""mujoco_warp_b200 -- H100-native (sm_90a) batched MuJoCo physics step behind the mujoco_warp API.

Public surface mirrors /root/reference/mujoco_warp/__init__.py for the step path: put_model, put_data, make_data,
reset_data, step, forward, the individually callable stages (with rne_postconstraint, subtree_vel, tendon, jac, xfrc_accumulate and
deriv_smooth_vel), potential and kinetic energy (energy_pos / energy_vel), actuator and sensor
delays (read_ctrl / read_sensor / init_ctrl_history / init_sensor_history), inverse
dynamics (inverse), ray casting (ray / rays), batch rendering (create_render_context, refit_bvh, render, get_rgb / get_depth /
get_segmentation) and the per-world recomputation of derived Model constants (set_const, set_const_fixed, set_const_0, set_const_spring,
set_length_range); `mjcf.load` stands in for mujoco's MJCF compiler.
"""

from . import scenes
from ._src import mjcf
from ._src._lib import build
from ._src.forward import camlight, collision, com_pos, crb, ctrl_noise, euler, factor_m, forward, fwd_acceleration, fwd_actuation
from ._src.forward import collision_kernel, fwd_position, fwd_velocity, kinematics, last_launch_count, make_constraint, solve, step, step_profile, team_residency, transmission
from ._src.forward import energy_pos, energy_vel
from ._src.forward import deriv_smooth_vel, jac, rne_postconstraint, subtree_vel, tendon, xfrc_accumulate
from ._src.forward import com_vel, contact_force, fwd_kinematics, get_state, implicit, mul_m, passive, rne, rungekutta4, sensor_acc, sensor_pos, sensor_vel, set_state, solve_m, step1, step2
from ._src.history import init_ctrl_history, init_sensor_history, read_ctrl, read_sensor
from ._src.inverse import inverse
from ._src.ray import ray, rays
from ._src.render import create_render_context, get_depth, get_rgb, get_segmentation, refit_bvh, render
from ._src.set_const import set_const, set_const_0, set_const_fixed, set_const_spring, set_length_range
from ._src.io import get_data_into, load_trajectory, make_data, override_model, put_data, put_model, reset_data, reset_data_keyframe
from ._src.trace import event_trace_step, flatten_trace
from ._src.types import BroadphaseFilter, BroadphaseType, ConeType, Constraint, ConstraintState, ConstraintType, Contact, Data
from ._src.types import BiasType, DynType, GainType, State, Statistic, TrnType
from ._src.types import DisableBit, EnableBit, GeomType, IntegratorType, JointType, Model, ObjType, Option, OverflowType, RenderContext, SolverType

__all__ = [n for n in dir() if not n.startswith("_")]
