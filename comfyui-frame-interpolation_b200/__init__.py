"""H100-native drop-in for the RIFE (and FILM, Sepconv, GMFSS Fortuna, FLAVR, IFRNet, CAIN, IFUnet) path of Fannovel16/ComfyUI-Frame-Interpolation (ComfyUI custom-node package).

Exports the same mapping names ComfyUI discovers in the reference's root __init__.py:23-47.
"""
from .node import RIFE_VFI, MakeInterpolationStateList, FloatToInt, InterpolationStateList  # noqa: F401
from .film_node import FILM_VFI  # noqa: F401
from .sepconv_node import SepconvVFI  # noqa: F401
from .gmfss_node import GMFSS_Fortuna_VFI  # noqa: F401
from .flavr_node import FLAVR_VFI  # noqa: F401
from .ifrnet_node import IFRNet_VFI  # noqa: F401
from .cain_node import CAIN_VFI  # noqa: F401
from .ifunet_node import IFUnet_VFI  # noqa: F401

NODE_CLASS_MAPPINGS = {
    "RIFE VFI": RIFE_VFI,
    "FILM VFI": FILM_VFI,
    "Sepconv VFI": SepconvVFI,
    "GMFSS Fortuna VFI": GMFSS_Fortuna_VFI,
    "FLAVR VFI": FLAVR_VFI,
    "IFRNet VFI": IFRNet_VFI,
    "CAIN VFI": CAIN_VFI,
    "IFUnet VFI": IFUnet_VFI,
    "Make Interpolation State List": MakeInterpolationStateList,
    "VFI FloatToInt": FloatToInt,
}

NODE_DISPLAY_NAME_MAPPINGS = {
    "RIFE VFI": "RIFE VFI (H100 native, rife4.6)",
    "FILM VFI": "FILM VFI (H100 native)",
    "Sepconv VFI": "Sepconv VFI (H100 native)",
    "GMFSS Fortuna VFI": "GMFSS Fortuna VFI (H100 native)",
    "FLAVR VFI": "FLAVR VFI (H100 native)",
    "IFRNet VFI": "IFRNet VFI (H100 native)",
    "CAIN VFI": "CAIN VFI (H100 native)",
    "IFUnet VFI": "IFUnet VFI (H100 native)",
}
