"""e4s_b200: the E4S synthesis hot path (mask-guided StyleGAN2 forward, inversion loop, RGI encoder) on hand-written sm_90a CUDA
behind a C ABI (include/e4s_b200.h).  See DESIGN.md."""


def set_deterministic(on: bool = True) -> None:
    """Ask for bit-reproducible tensor-core convolutions (on / off).  The forward kernels accumulate every output in a fixed
    order, so they are bit reproducible with either setting; the setting records the caller's requirement.  Also:
    environment E4S_B200_DETERMINISTIC=1."""
    from . import _lib
    _lib.check(_lib.load().e4s_set_deterministic(int(bool(on))), "e4s_set_deterministic")


def is_deterministic() -> bool:
    from . import _lib
    return bool(_lib.load().e4s_get_deterministic())


def invalidate_prepared(module) -> None:
    """Drop every cached kernel-ready weight form under `module` (bf16 operand planes, folded up-sampling kernels, stacked
    MLPs).  Needed only after in-place parameter writes that bypass autograd's version counter (``param.data.copy_()``, EMA
    accumulation loops); ``load_state_dict`` and ordinary in-place ops are detected automatically."""
    for m in module.modules():
        prep = getattr(m, "_prep", None)
        if hasattr(prep, "invalidate"):
            prep.invalidate()
        for attr in ("_prep_key", "_mlp_cache"):
            if hasattr(m, attr):
                setattr(m, attr, None)
        if hasattr(m, "_planes") and isinstance(m._planes, dict):
            m._planes.clear()
