"""`unicorn` — the reference's package name, served by unicorn_b200 (H100-native per-frame inference path).

Inference surface only: unicorn.exp.get_exp(...).get_model(), unicorn.utils.postprocess, unicorn.utils.boxes.postprocess_inst,
unicorn.tracker.{byte_tracker.BYTETracker, quasi_dense_embed_tracker.QuasiDenseEmbedTracker}, unicorn.models.Unicorn."""
__unicorn_b200_shim__ = True
__version__ = "0.1.0+b200"
