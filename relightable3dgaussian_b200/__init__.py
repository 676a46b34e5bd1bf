"""r3dg-b200: the Relightable3DGaussian renderer hot path on H100 (sm_90a).

Host mirrors of the reference's operator surface over one C-ABI CUDA library (include/r3dg_b200.h):
rasterizer (GaussianRasterizer), shading (rendering_equation), raytracer (RayTracer / visibility bake), optim
(FusedAdam, compaction), dist (view-parallel gradient exchange), formats (checkpoint / PLY / bake files).
Nothing is imported eagerly: `import relightable3dgaussian_b200` works without a GPU; the sub-modules load the
library on first use and raise if it is missing (there is no CPU fallback)."""
