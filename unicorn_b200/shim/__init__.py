"""`unicorn`-importable API shim (SURVEY.md 8b "Python model API to keep"; north_star: "keeping the unicorn.models / unicorn.tracker
Python API surface").  Put this directory FIRST on sys.path / PYTHONPATH and the reference's per-frame driver code
(external/lib/test/tracker/unicorn_sot.py, unicorn_vos.py, the per-frame bodies of unicorn/evaluators/mot_evaluator.py) resolves its
`unicorn.*` imports to the H100 path instead of the reference's PyTorch modules:

    import unicorn_b200.shim as shim; shim.install()        # or: PYTHONPATH=<repo>/unicorn_b200/shim
    from unicorn.exp import get_exp
    model = get_exp("exps/default/unicorn_track_large.py", None).get_model(load_pretrain=False)

Only the inference surface of the hot path exists here (see INTEGRATION.md); training, data loading and evaluators are out of scope."""
import os
import sys

PATH = os.path.dirname(os.path.abspath(__file__))


def install():
    """Make `import unicorn` resolve to this shim (idempotent).  Raises if another `unicorn` package is already imported."""
    mod = sys.modules.get("unicorn")
    if mod is not None and not getattr(mod, "__unicorn_b200_shim__", False):
        raise RuntimeError(f"a different `unicorn` package is already imported from {getattr(mod, '__file__', '?')}")
    if PATH not in sys.path:
        sys.path.insert(0, PATH)
    return PATH
