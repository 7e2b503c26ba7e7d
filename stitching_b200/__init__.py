"""stitching_b200 -- the compositing hot path of OpenStitching/stitching on NVIDIA H100 (sm_90a).

Drop-in replacements for `stitching.warper.Warper`, `stitching.blender.Blender` and `SeamFinder.resize` (same
interface) backed by hand-written CUDA kernels behind a C ABI (include/stitch_b200.h), plus a fused `Compositor`.
`install()` swaps them into an installed `stitching` package so that Stitcher / AffineStitcher / the CLI run
unchanged.
"""
from . import exposure_error_compensator, images, seam_finder  # noqa: F401
from .blender import Blender  # noqa: F401
from .compositor import Compositor, Crop  # noqa: F401
from .stitching_error import StitchingError, StitchingWarning  # noqa: F401
from .timelapser import Timelapser  # noqa: F401
from .warper import Warper  # noqa: F401

__version__ = "0.1.0"


_installed = {}


def install(stitching_module=None):
    """Route `stitching.Stitcher` (and cropper / seam finder / verbose callers) through the GPU classes.

    The reference modules bind the class names at import time (`from .warper import Warper` in
    stitcher.py, cropper.py, seam_finder.py, verbose.py), so the names are patched in each of them.  A reference
    module that cannot be imported is reported with a StitchingWarning (the pipeline would otherwise run half on cv2
    and half on the GPU classes without a sign); any other failure propagates.
    """
    import importlib
    import warnings

    if stitching_module is None:
        stitching_module = importlib.import_module("stitching")
    if _installed.get(id(stitching_module)) is stitching_module:
        return stitching_module
    pkg = stitching_module.__name__
    missing = []

    def module(name):
        try:
            return importlib.import_module(f"{pkg}.{name}")
        except ImportError as e:  # (ModuleNotFoundError included)
            missing.append(f"{pkg}.{name} ({e})")
            return None

    for mod, names in (
        ("warper", ("Warper",)), ("blender", ("Blender",)), ("timelapser", ("Timelapser",)),
        ("stitcher", ("Warper", "Blender", "Timelapser")),
        ("cropper", ("Blender",)), ("seam_finder", ("Blender",)), ("verbose", ("Warper", "Blender", "Timelapser")),
    ):
        m = module(mod)
        if m is None:
            continue
        for name in names:
            if hasattr(m, name):
                setattr(m, name, {"Warper": Warper, "Blender": Blender, "Timelapser": Timelapser}[name])
    # the FINAL-resolution step of the seam finder (seam_finder.py:38-43); stitcher.py calls it through the class
    sf = module("seam_finder")
    if sf is not None:
        sf.SeamFinder.resize = staticmethod(seam_finder.resize)
    # the resampling to MEDIUM / LOW / FINAL resolution (images.py:120-123)
    im = module("images")
    if im is not None:
        im.Images.resize_img_by_scaler = staticmethod(images.resize_img_by_scaler)
    # the FINAL-resolution step of the exposure compensator (exposure_error_compensator.py:43-45)
    ec = module("exposure_error_compensator")
    if ec is not None:

        def _apply(self, *args):
            return exposure_error_compensator.apply(self.compensator, *args)

        ec.ExposureErrorCompensator.apply = _apply
    if missing:
        warnings.warn("stitching_b200.install(): not patched, these stay on the reference's cv2 path: " + "; ".join(missing), StitchingWarning)
    _installed[id(stitching_module)] = stitching_module
    return stitching_module


def __getattr__(name):
    """`stitching_b200.Stitcher` / `stitching_b200.AffineStitcher` (stitching/__init__.py:1): the reference's pipeline
    classes -- same DEFAULT_SETTINGS, same CLI -- running on the GPU classes.  They live in the reference package
    (registration, seam estimation, cropping ... are its control plane); install() routes their hot path here."""
    if name in ("Stitcher", "AffineStitcher"):
        return getattr(install(), name)
    raise AttributeError(f"module 'stitching_b200' has no attribute {name!r}")
