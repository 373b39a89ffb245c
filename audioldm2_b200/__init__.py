"""Native (H100, sm_90a) AudioLDM2 sampling hot path.  Same top-level names as ``audioldm2/__init__.py:1-2``
(``from .utils import seed_everything, save_wave, get_time, get_duration, read_list`` and ``from .pipeline import *``)."""
from .utils import seed_everything, save_wave, get_time, get_duration, read_list      # noqa: F401
from .pipeline import (build_model, text_to_audio, super_resolution_and_inpainting,   # noqa: F401
                       style_transfer, round_up_duration,
                       make_batch_for_text_to_audio, wav_to_fbank, NativeAudioLDM2, SyntheticConditioning, select_best)

__all__ = ["seed_everything", "save_wave", "get_time", "get_duration", "read_list", "build_model", "text_to_audio",
           "super_resolution_and_inpainting", "style_transfer", "round_up_duration", "make_batch_for_text_to_audio",
           "wav_to_fbank", "NativeAudioLDM2", "SyntheticConditioning", "select_best"]
