"""Drop-in import surface of the reference package (ip_adapter/__init__.py:1-11).  SD1.5-only classes
(IPAdapter.generate, IPAdapterPlus, IPAdapterFull) are outside the SDXL hot path and are not provided."""
from .custom_pipelines import (StableDiffusionXLCustomPipeline, StableDiffusionXLImg2ImgPipeline,
                               StableDiffusionXLInpaintPipeline)
from .ip_adapter import AutoencoderTiny, IPAdapter, IPAdapterPlusXL, IPAdapterXL, MultiControlNetModel

__all__ = ["AutoencoderTiny", "IPAdapter", "IPAdapterPlusXL", "IPAdapterXL", "MultiControlNetModel", "StableDiffusionXLCustomPipeline",
           "StableDiffusionXLImg2ImgPipeline", "StableDiffusionXLInpaintPipeline"]
