"""ctypes binding of libr3dg_b200.so (C ABI: include/r3dg_b200.h).

There is NO fallback: if the CUDA library is missing or does not export a declared symbol this
module raises at import time, so a GPU run can never silently use anything but the sm_90a
kernels.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# R3DG_LIB_PATH: developer knob to load another build of the library (e.g. to A/B two builds); unset = the in-tree library
LIB_PATH = os.environ.get("R3DG_LIB_PATH") or os.path.join(_HERE, "libr3dg_b200.so")

c_void_p, c_int, c_float, c_size_t, c_ll = (ctypes.c_void_p, ctypes.c_int, ctypes.c_float,
                                            ctypes.c_size_t, ctypes.c_longlong)


class RasterFwdArgs(ctypes.Structure):
    _fields_ = (
        [(n, c_int) for n in ("P", "S", "D", "M", "W", "H")] +
        [(n, c_void_p) for n in ("background", "means3D", "shs", "colors_precomp", "features",
                                 "opacities", "scales", "rotations", "cov3D_precomp", "viewmatrix",
                                 "projmatrix", "campos")] +
        [(n, c_float) for n in ("scale_modifier", "tan_fovx", "tan_fovy", "cx", "cy")] +
        [(n, c_int) for n in ("prefiltered", "computer_pseudo_normal", "debug")] +
        [(n, c_void_p) for n in ("out_color", "out_opacity", "out_depth", "out_feature",
                                 "out_normal", "out_surface_xyz", "out_weights", "radii",
                                 "n_contrib")] +
        [("geom", c_void_p), ("geom_bytes", c_size_t), ("img", c_void_p), ("img_bytes", c_size_t),
         ("binning", c_void_p), ("binning_bytes", c_size_t), ("num_rendered_host", c_void_p), ("count_ready_event", c_void_p),
         ("V", c_int), ("view_cams", c_void_p), ("features_per_view", c_int), ("colors_per_view", c_int),
         ("filter_3d", c_void_p), ("depth_stats", c_int), ("out_depth2", c_void_p), ("out_median_depth", c_void_p),
         ("ray_depth", c_int), ("antialiasing", c_int),
         ("deterministic", c_int), ("det_work", c_void_p), ("det_work_bytes", c_size_t)])


class RasterBwdArgs(ctypes.Structure):
    _fields_ = (
        [(n, c_int) for n in ("P", "S", "D", "M", "W", "H")] +
        [(n, c_void_p) for n in ("background", "means3D", "shs", "colors_precomp", "features",
                                 "scales", "rotations", "cov3D_precomp", "viewmatrix",
                                 "projmatrix", "campos")] +
        [(n, c_float) for n in ("scale_modifier", "tan_fovx", "tan_fovy")] +
        [(n, c_int) for n in ("backward_geometry", "debug")] +
        [(n, c_void_p) for n in ("dL_dout_color", "dL_dout_opacity", "dL_dout_depth",
                                 "dL_dout_feature", "dL_dmeans2D", "dL_dcolors", "dL_dopacity",
                                 "dL_dmeans3D", "dL_dfeatures", "dL_dcov3D", "dL_dsh",
                                 "dL_dscales", "dL_drotations", "dL_dsh_factor")] +
        [("geom", c_void_p), ("geom_bytes", c_size_t), ("img", c_void_p), ("img_bytes", c_size_t),
         ("binning", c_void_p), ("binning_bytes", c_size_t),
         ("V", c_int), ("view_cams", c_void_p), ("features_per_view", c_int), ("colors_per_view", c_int),
         ("dL_dviewmatrix", c_void_p), ("dL_dprojmatrix", c_void_p), ("dL_dcampos", c_void_p),
         ("cam_work", c_void_p), ("cam_work_bytes", c_size_t),
         ("dL_dout_normal", c_void_p), ("dL_dout_surface_xyz", c_void_p), ("fwd_opacity", c_void_p), ("fwd_depth", c_void_p),
         ("cx", c_float), ("cy", c_float), ("surface_work", c_void_p), ("surface_work_bytes", c_size_t),
         ("filter_3d", c_void_p), ("opacities", c_void_p),
         ("depth_stats", c_int), ("dL_dout_depth2", c_void_p), ("dL_dout_median_depth", c_void_p),
         ("ray_depth", c_int), ("dL_dmeans2D_abs", c_void_p), ("antialiasing", c_int),
         ("deterministic", c_int), ("det_work", c_void_p), ("det_work_bytes", c_size_t)])


class ShadeArgs(ctypes.Structure):
    _fields_ = (
        [(n, c_int) for n in ("P", "N", "sh_coeffs", "env_h", "env_w")] +
        [(n, c_void_p) for n in ("base_color", "roughness", "normals", "viewdirs", "incidents", "env",
                                 "env_transform", "visibility", "incident_dirs", "incident_areas",
                                 "pbr", "diffuse_light", "specular", "mean_incident_lights",
                                 "mean_local_lights", "mean_global_lights", "mean_visibility",
                                 "incident_lights", "local_incident_lights", "global_incident_lights",
                                 "dL_dpbr", "dL_ddiffuse_light", "dL_dspecular", "dL_dbase_color",
                                 "dL_droughness", "dL_dviewdirs", "dL_dincidents", "dL_denv")] +
        [("V", c_int), ("transform_per_view", c_int), ("env_pyramid", c_void_p), ("dL_denv_pyramid", c_void_p)] +
        [("deterministic", c_int), ("det_work", c_void_p), ("det_work_bytes", c_size_t)])


class MultiviewArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("V", "H", "W", "B")] +
                [(n, c_void_p) for n in ("depth", "normal", "gray", "viewmatrix", "pair_cams", "pairs")] +
                [("pixel_noise_threshold", c_float)] +
                [(n, c_void_p) for n in ("geo", "photo", "counts", "work")] + [("work_bytes", c_size_t)] +
                [(n, c_void_p) for n in ("dL_dgeo", "dL_dphoto", "dL_ddepth", "dL_dnormal")] +
                [("deterministic", c_int), ("det_work", c_void_p), ("det_work_bytes", c_size_t)])


class LightArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("P", "K", "V")] +
                [(n, c_void_p) for n in ("kind", "vec", "color", "means3D", "base_color", "roughness", "normals", "viewdirs",
                                         "shadows", "pbr", "diffuse_light", "specular", "dL_dpbr", "dL_ddiffuse_light",
                                         "dL_dspecular", "dL_dbase_color", "dL_droughness", "dL_dviewdirs", "dL_dmeans3D",
                                         "dL_dvec", "dL_dcolor", "work")] +
                [("work_bytes", c_size_t)])


class ShapedLightArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("P", "K", "V", "M")] + [("seed", ctypes.c_uint32)] +
                [(n, c_void_p) for n in ("kind", "pos", "a", "b", "color", "cone", "means3D", "base_color", "roughness",
                                         "normals", "viewdirs", "shadows", "pbr", "diffuse_light", "specular", "dL_dpbr",
                                         "dL_ddiffuse_light", "dL_dspecular", "dL_dbase_color", "dL_droughness",
                                         "dL_dviewdirs", "dL_dmeans3D", "dL_dpos", "dL_da", "dL_db", "dL_dcolor",
                                         "dL_dcone", "work")] +
                [("work_bytes", c_size_t)])


class PixelArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("V", "H", "W", "N", "env_h", "env_w")] +
                [(n, c_void_p) for n in ("base_color", "roughness", "normal", "points", "campos", "incidents", "mask", "env",
                                         "env_transform")] +
                [("transform_per_view", c_int)] +
                [(n, c_void_p) for n in ("env_pyramid", "dL_denv_pyramid", "visibility", "pbr", "diffuse_light", "specular",
                                         "mean_visibility", "dL_dpbr", "dL_ddiffuse_light", "dL_dspecular", "dL_dbase_color",
                                         "dL_droughness", "dL_dincidents", "dL_denv")] +
                [("deterministic", c_int), ("det_work", c_void_p), ("det_work_bytes", c_size_t)] +
                [("sampler_table", c_void_p), ("n_env", c_int), ("n_ggx", c_int), ("seed", ctypes.c_uint32),
                 ("sampler_transform", c_void_p)])


class PixelLightArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("V", "H", "W", "K", "M")] + [("seed", ctypes.c_uint32)] +
                [(n, c_void_p) for n in ("kind", "pos", "a", "b", "color", "cone", "base_color", "roughness", "normal", "points",
                                         "campos", "mask", "shadows", "pbr", "diffuse_light", "specular", "dL_dpbr",
                                         "dL_ddiffuse_light", "dL_dspecular", "dL_dbase_color", "dL_droughness", "dL_dpos",
                                         "dL_da", "dL_db", "dL_dcolor", "dL_dcone", "work")] +
                [("work_bytes", c_size_t)])


class DenoiseArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("V", "H", "W", "C", "F", "L")] +
                [(n, c_float) for n in ("sigma_normal", "sigma_plane", "sigma_features")] +
                [(n, c_void_p) for n in ("normal", "points", "mask", "features", "x", "y", "dL_dy", "dL_dx", "work")] +
                [("work_bytes", c_size_t)])


class ComposeArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("P", "K")] +
                [(n, c_void_p) for n in ("offsets", "quat", "translation", "scale", "xyz", "normal", "rotation", "scaling")] +
                [("n_sh", c_int), ("sh_degree", c_int * 3), ("sh_channels", c_int * 3), ("sh", c_void_p * 3)] +
                [(n, c_void_p) for n in ("xyz_out", "normal_out", "rotation_out", "scaling_out")] + [("sh_out", c_void_p * 3)] +
                [(n, c_void_p) for n in ("dL_dxyz_out", "dL_dnormal_out", "dL_drotation_out", "dL_dscaling_out")] +
                [("dL_dsh_out", c_void_p * 3)] +
                [(n, c_void_p) for n in ("dL_dxyz", "dL_dnormal", "dL_drotation", "dL_dscaling")] + [("dL_dsh", c_void_p * 3)] +
                [(n, c_void_p) for n in ("dL_dR", "dL_dquat", "dL_dtranslation", "dL_dscale", "work")] +
                [("work_bytes", c_size_t)])


class TsdfIntegrateArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("NX", "NY", "NZ")] + [("origin", c_float * 3)] +
                [(n, c_float) for n in ("voxel_size", "sdf_trunc", "depth_trunc")] +
                [(n, c_void_p) for n in ("tsdf", "weight", "color")] + [(n, c_int) for n in ("V", "H", "W")] +
                [(n, c_void_p) for n in ("depth", "rgb", "viewmatrix", "cams")])


class TsdfExtractArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("NX", "NY", "NZ")] + [("origin", c_float * 3), ("voxel_size", c_float)] +
                [(n, c_void_p) for n in ("tsdf", "weight", "color", "work")] + [("work_bytes", c_size_t)] +
                [("totals_host", c_void_p), ("n_verts", c_ll), ("n_faces", c_ll)] +
                [(n, c_void_p) for n in ("verts", "vert_colors", "faces")])


class ExchangeArgs(ctypes.Structure):
    _fields_ = ([(n, c_int) for n in ("P", "D", "M", "world", "rank")] +
                [("means3D", c_void_p), ("campos", c_void_p), ("factors", c_void_p * 64), ("dL_dsh", c_void_p),
                 ("n_dense", c_ll), ("dense", c_void_p * 64), ("dense_multicast", c_void_p)])


class PackSrc(ctypes.Structure):
    _fields_ = [("ptr", c_void_p), ("width", c_int)]


class CompactTensor(ctypes.Structure):
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("row_bytes", c_ll)]


class DensifyTensor(ctypes.Structure):
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("row_bytes", c_ll), ("kind", c_int)]


class DensifyThresholds(ctypes.Structure):
    _fields_ = ([(n, c_float) for n in ("max_grad", "max_grad_normal", "dense_scale", "min_opacity", "weights_threshold",
                                        "max_screen_size", "big_scale", "split_recip")] +
                [("check_size", c_int)])


class AdamTensor(ctypes.Structure):
    _fields_ = ([(n, c_void_p) for n in ("param", "grad", "exp_avg", "exp_avg_sq")] +
                [("n", c_ll), ("step", c_ll)] +
                [(n, ctypes.c_double) for n in ("lr", "beta1", "beta2", "eps")] +
                [("row_mask", c_void_p), ("row_elems", c_ll)])


# every symbol include/r3dg_b200.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("r3dg_version", ctypes.c_char_p, []),
    ("r3dg_raster_geom_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_raster_img_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_raster_binning_bytes", c_size_t, [c_ll]),
    ("r3dg_raster_img_n_contrib_offset", c_size_t, [c_int, c_int]),
    ("r3dg_raster_views_geom_bytes", c_size_t, [c_int, c_int, c_int]),
    ("r3dg_raster_views_img_bytes", c_size_t, [c_int, c_int, c_int]),
    ("r3dg_raster_views_img_n_contrib_offset", c_size_t, [c_int, c_int, c_int]),
    ("r3dg_raster_ray_depth_geom_bytes", c_size_t, [c_int, c_int, c_int]),
    ("r3dg_raster_depth_stats_img_bytes", c_size_t, [c_int, c_int, c_int]),
    ("r3dg_raster_forward", c_int, [ctypes.POINTER(RasterFwdArgs), c_void_p]),
    ("r3dg_raster_backward", c_int, [ctypes.POINTER(RasterBwdArgs), c_void_p]),
    ("r3dg_raster_cam_grad_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_raster_surface_grad_bytes", c_size_t, [c_int, c_int, c_int]),
    ("r3dg_sh_grad_from_factors", c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p]),
    ("r3dg_exchange_p2p", c_int, [ctypes.POINTER(ExchangeArgs), c_void_p]),
    ("r3dg_mark_visible", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_bvh_build_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_bvh_trace_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_bvh_leaf_aabbs", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_bvh_build", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("r3dg_bvh_trace_opacity", c_int, [c_int, c_ll, c_void_p, c_void_p, c_void_p, c_int, c_float, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_size_t, c_void_p]),
    ("r3dg_sample_incident_dirs", c_int, [c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_bvh_bake_visibility", c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("r3dg_bvh_bake_radiance_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_bvh_bake_radiance", c_int, [c_int, c_int] + [c_void_p] * 7 + [c_int, c_int, c_float] + [c_void_p] * 4 +
                                      [c_size_t, c_void_p]),
    ("r3dg_fit_incident_sh", c_int, [c_int, c_int, c_void_p, c_void_p, c_int, c_float, c_void_p, c_void_p]),
    ("r3dg_bvh_trace_lights_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_bvh_trace_lights", c_int, [c_int, c_int] + [c_void_p] * 9 + [c_void_p, c_size_t, c_void_p]),
    ("r3dg_shade_lights_work_bytes", c_size_t, [c_int, c_int]),
    # `const struct r3dg_light_args*`: pass ctypes.byref(LightArgs(...))
    ("r3dg_shade_lights_forward", c_int, [c_void_p, c_void_p]),
    ("r3dg_shade_lights_backward", c_int, [c_void_p, c_void_p]),
    ("r3dg_shaped_lights_num_rays", c_int, [c_int, c_void_p, c_int]),
    ("r3dg_bvh_trace_shaped_lights_tmp_bytes", c_size_t, [c_int]),
    # `const struct r3dg_shaped_light_args*`: pass ctypes.byref(ShapedLightArgs(...))
    ("r3dg_bvh_trace_shaped_lights", c_int, [c_void_p] * 7 + [c_size_t, c_void_p]),
    ("r3dg_shade_shaped_lights_work_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_shade_shaped_lights_forward", c_int, [c_void_p, c_void_p]),
    ("r3dg_shade_shaped_lights_backward", c_int, [c_void_p, c_void_p]),
    ("r3dg_bvh_trace_pixels_tmp_bytes", c_size_t, [c_int]),
    # `const struct r3dg_pixel_args*`: pass ctypes.byref(PixelArgs(...))
    ("r3dg_bvh_trace_pixels", c_int, [c_void_p, c_int] + [c_void_p] * 8 + [c_size_t, c_void_p]),
    ("r3dg_shade_pixels_forward", c_int, [c_void_p, c_void_p]),
    ("r3dg_shade_pixels_backward", c_int, [c_void_p, c_void_p]),
    ("r3dg_bvh_trace_pixel_lights_tmp_bytes", c_size_t, [c_int]),
    # `const struct r3dg_pixel_light_args*`: pass ctypes.byref(PixelLightArgs(...))
    ("r3dg_bvh_trace_pixel_lights", c_int, [c_void_p, c_int] + [c_void_p] * 8 + [c_size_t, c_void_p]),
    ("r3dg_shade_pixel_lights_work_bytes", c_size_t, [c_int, c_int, c_int, c_int]),
    ("r3dg_shade_pixel_lights_forward", c_int, [c_void_p, c_void_p]),
    ("r3dg_shade_pixel_lights_backward", c_int, [c_void_p, c_void_p]),
    ("r3dg_denoise_work_bytes", c_size_t, [c_int] * 6),
    # `const struct r3dg_denoise_args*`: pass ctypes.byref(DenoiseArgs(...))
    ("r3dg_denoise_forward", c_int, [c_void_p, c_void_p]),
    ("r3dg_denoise_backward", c_int, [c_void_p, c_void_p]),
    ("r3dg_compose_work_bytes", c_size_t, [c_int, c_int]),
    # `const struct r3dg_compose_args*`: pass ctypes.byref(ComposeArgs(...))
    ("r3dg_compose_forward", c_int, [c_void_p, c_void_p]),
    ("r3dg_compose_backward", c_int, [c_void_p, c_void_p]),
    ("r3dg_unpremultiply_forward", c_int, [c_int, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_unpremultiply_backward", c_int, [c_int, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_render_equation_forward", c_int, [ctypes.POINTER(ShadeArgs), c_void_p]),
    ("r3dg_render_equation_backward", c_int, [ctypes.POINTER(ShadeArgs), c_void_p]),
    ("r3dg_env_pyramid_levels", c_int, [c_int, c_int]),
    ("r3dg_env_pyramid_floats", c_size_t, [c_int, c_int]),
    ("r3dg_env_pyramid_build", c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    ("r3dg_shade_filtered_det_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_env_sampler_floats", c_size_t, [c_int, c_int]),
    ("r3dg_env_sampler_build", c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    ("r3dg_sample_importance_dirs", c_int, [c_int, c_int] + [c_void_p] * 5 + [c_int, c_int, ctypes.c_ulonglong] +
                                           [c_void_p, c_void_p, c_void_p]),
    ("r3dg_pack_features_forward", c_int, [c_int, c_int, c_void_p, c_void_p, c_int, ctypes.POINTER(PackSrc), c_void_p, c_void_p]),
    ("r3dg_pack_features_backward", c_int, [c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, ctypes.POINTER(PackSrc), c_void_p,
                                            c_void_p, c_void_p, c_size_t, c_void_p]),
    ("r3dg_compact_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_compact_scan", c_int, [c_int, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    ("r3dg_compact_rows", c_int, [c_int, c_int, ctypes.POINTER(CompactTensor), c_void_p, c_void_p, c_void_p]),
    ("r3dg_densify_stats", c_int, [c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_densify_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_densify_classify", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      ctypes.POINTER(DensifyThresholds), c_void_p, c_size_t, c_void_p, c_void_p]),
    ("r3dg_densify_apply", c_int, [c_int, ctypes.POINTER(c_int), c_int, ctypes.POINTER(DensifyTensor), c_void_p, c_void_p,
                                   c_void_p, c_float, c_void_p, c_size_t, c_void_p]),
    ("r3dg_mcmc_tmp_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_mcmc_noise", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_double, ctypes.c_double,
                                ctypes.c_double, c_void_p]),
    ("r3dg_mcmc_classify", c_int, [c_int, c_void_p, c_float, c_void_p, c_size_t, c_void_p]),
    ("r3dg_mcmc_apply", c_int, [c_int, c_int, c_void_p, c_void_p, c_void_p, ctypes.c_double, c_int, c_int,
                                ctypes.POINTER(DensifyTensor), c_void_p, c_size_t, c_void_p]),
    ("r3dg_filter3d_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_filter3d_compute", c_int, [c_int, c_int, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_size_t,
                                      c_void_p]),
    ("r3dg_raster_fwd_det_bytes", c_size_t, [c_int]),
    ("r3dg_raster_bwd_det_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_raster_ray_depth_bwd_det_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_raster_bwd_det_absgrad_bytes", c_size_t, [c_int]),
    ("r3dg_shade_det_bytes", c_size_t, [c_int, c_int]),
    ("r3dg_det_sum_host", c_int, [c_ll, c_void_p, c_void_p]),
    ("r3dg_det_sum_scaled_host", c_int, [c_ll, c_void_p, c_float, c_void_p]),
    ("r3dg_knn_tmp_bytes", c_size_t, [c_int]),
    ("r3dg_knn_dist2", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("r3dg_ssim_tmp_bytes", c_size_t, [c_int, c_int, c_int, c_int]),
    ("r3dg_ssim_forward", c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("r3dg_ssim_backward", c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    ("r3dg_edge_aware_tmp_bytes", c_size_t, [c_int, c_int, c_int, c_int]),
    ("r3dg_edge_aware_forward", c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("r3dg_edge_aware_backward", c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_tv_tmp_bytes", c_size_t, [c_int, c_int, c_int]),
    ("r3dg_tv_forward", c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("r3dg_tv_backward", c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("r3dg_bilagrid_tmp_bytes", c_size_t, [c_int] * 7),
    ("r3dg_bilagrid_forward", c_int, [c_int] * 7 + [c_void_p] * 5),
    ("r3dg_bilagrid_backward", c_int, [c_int] * 7 + [c_void_p] * 7 + [c_size_t, c_void_p]),
    ("r3dg_multiview_work_bytes", c_size_t, [c_int] * 3),
    ("r3dg_multiview_det_bytes", c_size_t, [c_int] * 3),
    # `const struct r3dg_multiview_args*`: pass ctypes.byref(MultiviewArgs(...))
    ("r3dg_multiview_forward", c_int, [c_void_p, c_void_p]),
    ("r3dg_multiview_backward", c_int, [c_void_p, c_void_p]),
    ("r3dg_tsdf_extract_work_bytes", c_size_t, [c_int] * 3),
    # `const struct r3dg_tsdf_*_args*`: pass ctypes.byref(TsdfIntegrateArgs(...)) / ctypes.byref(TsdfExtractArgs(...))
    ("r3dg_tsdf_integrate", c_int, [c_void_p, c_void_p]),
    ("r3dg_tsdf_extract_count", c_int, [c_void_p, c_void_p]),
    ("r3dg_tsdf_extract_emit", c_int, [c_void_p, c_void_p]),
    ("r3dg_adam_step", c_int, [c_int, ctypes.POINTER(AdamTensor), c_void_p]),
    ("r3dg_launch_count", ctypes.c_ulonglong, []),
    ("r3dg_tune", c_int, [ctypes.c_char_p, c_int, ctypes.POINTER(c_int)]),
    ("r3dg_prof_begin", c_int, [c_int]),
    ("r3dg_prof_end", c_int, [ctypes.POINTER(c_float), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    ("r3dg_raster_debug_copy", c_ll, [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_size_t, c_void_p, c_ll, c_void_p]),
    ("r3dg_raster_ray_depth_debug_copy", c_ll, [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_size_t, c_void_p, c_ll, c_void_p]),
]

_lib = None


def load():
    """Load the library and bind every declared symbol.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found — build it with `python -m relightable3dgaussian_b200.build` "
            "(there is no CPU/PyTorch fallback for the rasterizer hot path)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(lib, name)      # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def tune(key, value):
    """Set a tuning knob (include/r3dg_b200.h: r3dg_tune); returns the previous value."""
    prev = c_int(0)
    check(load().r3dg_tune(key.encode(), int(value), ctypes.byref(prev)), f"r3dg_tune({key})")
    return prev.value


def check(rc, what):
    if rc != 0:
        if rc in (-10001, -10002):
            raise RuntimeError(f"{what}: {'bad argument' if rc == -10001 else 'unsupported configuration'} ({rc})")
        raise RuntimeError(f"{what}: CUDA error {-rc}")


def call(name, device, *args, what=None):
    """Run the launching entry point `name` on `device`, enqueued on torch's current stream of that device (every
    launching entry point takes the stream last); a non-zero status raises through check() with `what`."""
    with torch.cuda.device(device):
        check(getattr(load(), name)(*args, torch.cuda.current_stream(device).cuda_stream), what or name)


def scratch(nbytes, device):
    """Uninitialised device workspace of `nbytes` bytes."""
    return torch.empty((nbytes,), dtype=torch.uint8, device=device)


def ptr(t):
    """Device pointer of an optional tensor; empty tensors mean "absent" (NULL), like the
    reference (forward.cu:206,242)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def f32(t):
    """`t` detached from autograd as a contiguous float32 tensor (the same storage when it already is one)."""
    return t.detach().float().contiguous()


def aligned16(t):
    """`t` itself when its data is 16-byte aligned (or it is absent / empty), else an aligned contiguous copy.  The
    library reads quaternions as float4 and refuses a misaligned `rotations`, such as a contiguous view at a storage
    offset that is not a multiple of 4 floats."""
    if t is None or t.numel() == 0 or t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=torch.contiguous_format)


def det_workspace(args, nbytes, device):
    """Under torch.are_deterministic_algorithms_enabled(), read at call time: a workspace of `nbytes` for the
    library's deterministic mode, entered into the argument struct `args` (deterministic, det_work, det_work_bytes).
    Otherwise None, and `args` keeps the default mode.  The caller holds the workspace until the call is enqueued."""
    if not torch.are_deterministic_algorithms_enabled():
        return None
    ws = scratch(nbytes, device)
    args.deterministic, args.det_work, args.det_work_bytes = 1, ws.data_ptr(), ws.numel()
    return ws
