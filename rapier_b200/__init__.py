"""rapier_b200 -- H100-native (sm_90a) step hot path behind Rapier's API (see DESIGN.md)."""
from . import _abi  # noqa: F401
from .sets import (ColliderBuilder, ColliderSet, FixedJointBuilder, ImpulseJointSet, RigidBodyBuilder,  # noqa: F401
                   RigidBodySet, SphericalJointBuilder, SpringJointBuilder, RopeJointBuilder)
