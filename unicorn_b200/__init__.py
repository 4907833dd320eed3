"""unicorn_b200 — H100-native (sm_90a) implementation of Unicorn's per-frame inference hot path."""
__version__ = "0.1.0"
