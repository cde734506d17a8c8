"""d9d_b200 — a Hopper (H100, sm_90a) native distributed-training framework with the capabilities of d9d."""

__version__ = "0.1.0"
