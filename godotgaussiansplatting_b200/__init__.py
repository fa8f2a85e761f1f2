"""gsr -- H100-native forward 3D-Gaussian-splatting rasterizer (drop-in for the hot path of
2Retr0/GodotGaussianSplatting's util/gaussian_splatting_rasterizer.gd)."""
__version__ = "0.1.0"
