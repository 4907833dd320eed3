"""Drop-in for the reference's native extension module `MultiScaleDeformableAttention`
(unicorn/models/ops/src/vision.cpp:13-16; imported at unicorn/models/ops/functions/ms_deform_attn_func.py:18).

Put this directory on sys.path (or call unicorn_b200.compat.install()) and the reference's `MSDeformAttnFunction`
runs unmodified on the sm_90a kernel `uc_msda_forward_f32`.  Same contract as the reference op
(ops/src/cuda/ms_deform_attn_cuda.cu:20-80): contiguous CUDA tensors, value [B,S,M,D], spatial_shapes [L,2] int64,
level_start_index [L] int64, sampling_loc [B,Lq,M,L,P,2], attn_weight [B,Lq,M,L,P]; returns a new [B,Lq,M*D] tensor.
CPU tensors raise (the reference's CPU stub also only raises, ops/src/cpu/ms_deform_attn_cpu.cpp:17-40)."""

from unicorn_b200 import ops


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
    for name, t in (("value", value), ("spatial_shapes", spatial_shapes), ("level_start_index", level_start_index),
                    ("sampling_loc", sampling_loc), ("attn_weight", attn_weight)):
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor (Not implemented on the CPU)")
        if not t.is_contiguous():
            raise RuntimeError(f"{name} tensor has to be contiguous")
    batch = value.shape[0]
    step = min(batch, int(im2col_step))
    if batch % step != 0:
        raise RuntimeError(f"batch({batch}) must divide im2col_step({step})")
    dt = value.dtype
    out = ops.msda_forward(value.float(), spatial_shapes.long(), level_start_index.long(), sampling_loc.float(), attn_weight.float())
    return out.to(dt)


def ms_deform_attn_backward(*args, **kwargs):
    raise NotImplementedError("unicorn_b200 implements the inference path only (MSDA backward is training-side, SURVEY §8a a6)")
