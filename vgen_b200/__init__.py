"""vgen_b200 -- H100-native (sm_90a) implementation of the VGen sampling hot path:
DiffusionDDIM.ddim_sample_loop -> UNetSD_T2VBase / UNetSD_I2VGen (and the VideoLCM / TF-T2V / DreamVideo / InstructVideo
LoRA / SR600 / HiGen variants, with the VideoComposer condition encoders and the DreamVideo adapters) forward ->
AutoencoderKL.decode, exposed under the reference's MODEL / DIFFUSION / AUTO_ENCODER registry names (`register()`), and
the VideoComposer engines' depth annotator (`MiDaS` / `midas_v3`), sketch annotators (`PiDiNet` / `pidinet_bsd`,
`SketchSimplification` / `sketch_simplification_gan`), canny annotator (`CannyDetector`, `canny_video`) and colour-palette
annotator (`Palette`, `histogram_video`), and DreamVideo's textual-inversion text path
(`FrozenOpenCLIPCustomEmbedder` + `EmbeddingManager`, EMBEDDER / EMBEDMANAGER) with DDIM inversion
(`DiffusionDDIM.ddim_reverse_sample_loop`), and DreamVideo's evaluation metric (`calculate_metric`, `score_video`,
`load_clip`, `dino_transform`, with the DINO ViT `vit_small`), and InstructVideo's segmental HPSv2 reward
(`SegmentalReward`, `load_hps`, `segment_indices`).

Every op of the path is a hand-written CUDA kernel in libvgen_b200.so (include/vgen_b200.h); this
package holds only the host-side mirror of the reference interface.  There is no CPU / PyTorch
fallback: without the built library or a CUDA device the forward raises.
"""
from .registry import register  # noqa: F401


def __getattr__(name):  # lazy: importing the package must not require torch.cuda
    if name in ("UNetSD_T2VBase", "UNetSD_I2VGen", "UNetSD_VideoLCM", "UNetSD_TFT2V", "UNetSD_DreamVideo", "UNetSD_LoRA",
                "UNetSD_SR600", "UNetSD_HiGen"):
        from . import unet
        return getattr(unet, name)
    if name == "AutoencoderKL":
        from .autoencoder import AutoencoderKL
        return AutoencoderKL
    if name in ("DiffusionDDIM", "DiffusionDDIMReward"):
        from . import diffusion
        return getattr(diffusion, name)
    if name in ("GaussianDiffusion", "DiffusionDDIMSR"):
        from . import diffusion_gauss
        return getattr(diffusion_gauss, name)
    if name in ("FrozenOpenCLIPEmbedder", "FrozenOpenCLIPVisualEmbedder", "FrozenOpenCLIPTextVisualEmbedder",
                "FrozenOpenCLIPEmbedderZero", "FrozenOpenCLIPCustomEmbedder"):
        from . import clip
        return getattr(clip, name)
    if name == "EmbeddingManager":
        from .embedding_manager import EmbeddingManager
        return EmbeddingManager
    if name in ("MiDaS", "midas_v3"):
        from . import depth
        return getattr(depth, name)
    if name in ("PiDiNet", "pidinet_bsd", "SketchSimplification", "sketch_simplification_gan"):
        from . import sketch
        return getattr(sketch, name)
    if name in ("calculate_metric", "score_video", "load_clip", "dino_transform"):
        from . import metric
        return getattr(metric, name)
    if name in ("CannyDetector", "canny_video"):
        from . import canny
        return getattr(canny, name)
    if name in ("Palette", "histogram_video"):
        from . import palette
        return getattr(palette, name)
    if name in ("SegmentalReward", "load_hps", "segment_indices"):
        from . import reward
        return getattr(reward, name)
    if name in ("vit_tiny", "vit_small", "vit_base"):
        from . import dino
        return getattr(dino, name)
    if name == "LCMScheduler":
        from .lcm import LCMScheduler
        return LCMScheduler
    raise AttributeError(name)
