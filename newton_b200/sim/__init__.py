from .articulation import (  # noqa: F401
    eval_fk, eval_ik, eval_inverse_dynamics_force, eval_inverse_dynamics_passive, eval_jacobian, eval_mass_matrix,
)
from .builder import JointDofConfig, ModelBuilder, ShapeConfig
from .enums import MAXVAL, BodyFlags, GeoType, JointType, ModelFlags, ShapeFlags, StateFlags
from .model import Contacts, Control, Model, State

__all__ = [
    "MAXVAL", "BodyFlags", "Contacts", "Control", "GeoType", "JointDofConfig", "JointType", "Model",
    "ModelBuilder", "ModelFlags", "ShapeConfig", "ShapeFlags", "State", "StateFlags", "eval_fk", "eval_ik",
    "eval_jacobian", "eval_mass_matrix", "eval_inverse_dynamics_passive", "eval_inverse_dynamics_force",
]
