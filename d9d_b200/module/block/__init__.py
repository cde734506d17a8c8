"""Neural building blocks. Every block runs its hot ops through ``d9d_b200.kernel`` (native sm_90a on CUDA)."""
