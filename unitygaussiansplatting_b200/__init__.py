"""H100-native Gaussian-splat render path behind the GaussianSplatRenderer / GaussianSplatAsset API
of aras-p/UnityGaussianSplatting.  The product is libgsplat_b200.so (CUDA, sm_90a) behind the C ABI
in include/gsplat_b200.h; this package is the thin host-side mirror used by tests and bench."""
from .asset import (ColorFormat, GaussianSplatAsset, SHFormat, VectorFormat, QUALITY, SCENE_CLUSTERED, SCENE_LATTICE,
                    SCENE_UNIFORM, create_asset, generate_input_splats, load_asset, read_ply, read_spz, save_asset, synthetic_asset, write_ply)
from .camera import Camera, look_rotation, trs, quat_to_mat
from .renderer import (GaussianSplatContext, GaussianSplatRenderer, GatherSplatsForCamera, SortAndRenderSplatsMulti,
                       make_frame_params)
from .pack import pack_asset
from ._native import GsError

__all__ = ["ColorFormat", "GaussianSplatAsset", "SHFormat", "VectorFormat", "QUALITY", "SCENE_CLUSTERED", "SCENE_LATTICE",
           "SCENE_UNIFORM", "create_asset", "generate_input_splats", "read_ply", "read_spz", "write_ply", "save_asset", "load_asset", "synthetic_asset", "Camera", "look_rotation", "trs",
           "quat_to_mat", "GaussianSplatContext", "GaussianSplatRenderer", "GatherSplatsForCamera", "SortAndRenderSplatsMulti", "make_frame_params", "pack_asset", "GsError"]
