"""cycle_diffusion_b200 -- H100-native CycleDiffusion sampling engine (DPM-Encoder inversion + guided decode).

Import order matters only in that `_cabi` loads libcdx.so eagerly: a missing library is an ImportError, never a
silent fallback.  `specs` is importable without the library (pure inventories / synthetic weights).
"""
__all__ = ['specs']
