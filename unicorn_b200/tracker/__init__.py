from .quasi_dense import QuasiDenseEmbedTracker, bdd_tracker  # noqa: F401
from .byte_tracker import BYTETracker  # noqa: F401
