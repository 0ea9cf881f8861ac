"""igneous_b200 -- H100-native (sm_90a) implementation of the igneous
per-chunk hot path: DownsampleTask pooling, 6-connected CCL, MeshTask
marching cubes, behind igneous's own task API.

Importing this package never touches the GPU; the native library is loaded on
first use (`igneous_b200._shim.load()`), and compute calls raise if it or a
CUDA device is missing -- there is no CPU fallback.
"""
__version__ = "0.1.0"


# The import surface of igneous/__init__.py:1-4 (`from igneous import DownsampleTask, MeshTask,
# Mesher, LocalTaskQueue, CloudVolume ...`, used by test/test_tasks.py:18-23), resolved lazily so
# that importing the package stays free of side effects (no native library, no storage layer).
_TASK_NAMES = ("DownsampleTask", "TransferTask", "ImageShardTransferTask", "ImageShardDownsampleTask", "CCLFacesTask", "CCLEquivalancesTask", "RelabelCCLTask",
               "create_relabeling", "clean_intermediate_files", "MeshTask", "downsample_and_upload",
               "downsample_method_to_fn", "threshold_image", "blackout_non_face_rails", "DisjointSet",
               "QuantizeTask", "CLAHETask", "ContrastNormalizationTask", "LuminanceLevelsTask",
               "SpatialIndexTask", "CountVoxelsTask", "SkeletonTask", "UnshardedSkeletonMergeTask",
               "BlackoutTask", "TouchTask", "DeleteTask", "ShardedFromUnshardedSkeletonMergeTask",
               "MeshManifestPrefixTask", "MeshManifestFilesystemTask", "TransferMeshFilesTask", "DeleteMeshFilesTask",
               "TransferSkeletonFilesTask", "DeleteSkeletonFilesTask")
# creators whose task is in _TASK_NAMES and that have no other root-level name in the reference
_CREATION_NAMES = ("create_sharded_skeletons_from_unsharded_tasks", "create_mesh_manifest_tasks",
                   "create_mesh_deletion_tasks", "create_xfer_meshes_tasks", "create_skeleton_deletion_tasks",
                   "create_xfer_skeleton_tasks")
_COMPAT_NAMES = ("CloudVolume", "EmptyVolumeException", "LocalTaskQueue", "RegisteredTask", "queueable")
__all__ = ["Mesher", "__version__"] + list(_TASK_NAMES) + list(_CREATION_NAMES) + list(_COMPAT_NAMES)


def __getattr__(name):
  if name == "Mesher":
    from .zmesh import Mesher
    return Mesher
  if name in _TASK_NAMES:
    from . import tasks
    return getattr(tasks, name)
  if name in _CREATION_NAMES:
    from . import task_creation
    return getattr(task_creation, name)
  if name in _COMPAT_NAMES:
    from . import _compat
    return getattr(_compat, name)
  raise AttributeError("module 'igneous_b200' has no attribute %r" % name)
