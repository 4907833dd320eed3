"""unicorn.models — `Unicorn` is the H100 model facade (reference: unicorn/models/unicorn.py:28-139, inference modes only)."""
from unicorn_b200.compat.model import UnicornB200Model as Unicorn  # noqa: F401
