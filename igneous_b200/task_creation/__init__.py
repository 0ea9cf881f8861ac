from .common import (FinelyDividedTaskIterator, get_bounds, num_tasks, operator_contact,
                     compute_shard_params_for_hashed)
from .image import (create_downsampling_tasks, create_image_shard_downsample_tasks, create_transfer_tasks,
                    create_transfer_cloudvolume, clean_xfer_info, _select_compression_by_encoding,
                    create_image_shard_transfer_tasks, num_mips_from_memory_target, create_ccl_face_tasks,
                    create_ccl_equivalence_tasks, create_ccl_relabel_tasks, MEMORY_TARGET,
                    create_contrast_normalization_tasks, create_luminance_levels_tasks, create_clahe_tasks,
                    create_quantized_affinity_info, create_quantize_tasks, create_voxel_counting_tasks,
                    create_blackout_tasks, create_touch_tasks, create_deletion_tasks, compute_rois)
from .mesh import create_meshing_tasks, create_spatial_index_mesh_tasks
from .skeleton import (create_skeletonizing_tasks, create_spatial_index_skeleton_tasks,
                       create_unsharded_skeleton_merge_tasks, create_sharded_skeletons_from_unsharded_tasks)
from ..tasks import ShardedFromUnshardedSkeletonMergeTask  # noqa: F401  (next to its creator)
