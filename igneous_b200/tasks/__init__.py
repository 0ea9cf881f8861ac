from .image import (DownsampleTask, TransferTask, ImageShardTransferTask, ImageShardDownsampleTask, downsample_and_upload,
                    downsample_method_to_fn, QuantizeTask, CLAHETask, ContrastNormalizationTask,
                    LuminanceLevelsTask, CountVoxelsTask, BlackoutTask, TouchTask, DeleteTask)
from .ccl import (CCLFacesTask, CCLEquivalancesTask, RelabelCCLTask, create_relabeling,
                  clean_intermediate_files, threshold_image, blackout_non_face_rails, DisjointSet)
from .mesh import MeshTask
from .spatial_index import SpatialIndexTask
from .skeleton import SkeletonTask, UnshardedSkeletonMergeTask, ShardedFromUnshardedSkeletonMergeTask
