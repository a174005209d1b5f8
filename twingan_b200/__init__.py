"""twingan_b200 -- H100-native (sm_90a) engine for the TwinGAN G+D training step and the
inference-only generator of jerryli27/TwinGAN.  See DESIGN.md.

Layout: csrc/ (CUDA kernels + the C-ABI of include/twg.h, built into libtwg.so), `ops` (operator
layer over the C-ABI), `pggan_utils` / `pggan` / `twingan` (host-side mirrors of the reference's
nets/pggan_utils.py, nets/pggan.py, twingan.py + image_generation.py losses/optimisation).
"""
__version__ = '0.1.0'
