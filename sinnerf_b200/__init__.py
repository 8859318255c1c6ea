"""sinnerf_b200 -- Hopper (sm_90a, H100) volumetric renderer behind SinNeRF's render_rays /
NeRF / Embedding interface.  See DESIGN.md and INTEGRATION.md."""
from .config import get_precision, set_precision, get_train_storage, set_train_storage  # noqa: F401

__version__ = "0.1.0"


def __getattr__(name):
    # torch-dependent modules are imported lazily so `import sinnerf_b200.build` stays light
    if name in ("render_rays", "render_rays_multi", "sample_pdf", "eval_points", "RayLosses"):
        from . import rendering
        return getattr(rendering, name)
    if name in ("NeRF", "Embedding"):
        from . import nerf
        return getattr(nerf, name)
    if name in ("FusedAdam", "FusedSGD", "FusedRAdam", "FusedRanger", "get_optimizer"):
        from . import optim
        return getattr(optim, name)
    if name == "forward_warp":
        from . import warp
        return warp.forward_warp
    raise AttributeError(name)
