# hot-path members of morefusion/contrib/__init__.py:3-11
from .iterative_closest_point_link import IterativeClosestPointLink  # noqa: F401
from .iterative_collision_check_link import IterativeCollisionCheckLink  # noqa: F401
from .iterative_collision_check_link import LossObserver  # noqa: F401  (ros/.../collision_based_pose_refinement.py:18)
from . import singleview_3d  # noqa: F401
from . import singleview_pcd  # noqa: F401
from .occupancy_registration import OccupancyRegistration  # noqa: F401  (SURVEY.md 8f-4)
from .multi_instance_octree_mapping import MultiInstanceOctreeMapping  # noqa: F401  (SURVEY.md 8f-3)
from .object_mapping import ObjectMapping  # noqa: F401  (ros/.../nodes/object_mapping.py)
from .icp_registration import ICPRegistration  # noqa: F401  (ros/.../singleview_3d_pose_estimation.py:246-264)
from .picking_order import SelectPickingOrder  # noqa: F401  (ros/.../nodes/select_picking_order.py)
