"""pyramid_flow_b200 — H100-native kernels behind the Pyramid-Flow sampler hot path (DiT step + causal-VAE decode).

Only what the hot path needs lives here: `csrc/` (sm_90a CUDA kernels + the C-ABI), `_lib`/`ops` (ctypes binding),
and the host-side mirrors of the reference interfaces (`dit`, `vae`, `scheduler`).
"""
__all__ = ["_lib", "ops"]
