"""monoport_b200 -- H100-native (sm_90a) occupancy-field hot path of MonoPort.

Public surface (mirrors the reference's, see INTEGRATION.md):
    monoport_b200.modeling.MonoPortNet / PIFuNetG / PIFuNetC     (monoport/lib/modeling/MonoPortNet.py)
    monoport_b200.modeling.geometry.{index, orthogonal, perspective}
    monoport_b200.engine.{Seg3dLossless, Seg3dTopk}              (implicit_seg.functional)
    monoport_b200.recon.{pifu_calib, forward_vertices, reconstruction, marching_cubes}
    monoport_b200.shard.{slab_bounds, query_grid_sharded}        (z-slab sharding over GPUs)
    monoport_b200.pipeline.FramePipeline                         (frame overlap for `processors=[...]` style pipelines)
    monoport_b200.mesh_util.{save_obj_mesh, save_obj_mesh_with_color}
The top-level packages `monoport/` and `implicit_seg/` of this repo re-export these under the reference's
import paths so RTL/main.py's imports resolve unchanged.
"""
__version__ = "0.1.0"
