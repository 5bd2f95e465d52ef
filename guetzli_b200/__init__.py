"""guetzli_b200: H100-native (sm_90a) implementation of Guetzli's hot path
behind Guetzli's own API surface.  See DESIGN.md / INTEGRATION.md.

    from guetzli_b200 import Params, ProcessStats, process, butteraugli_score_for_quality
    params = Params(butteraugli_target=butteraugli_score_for_quality(95))
    ok, jpeg = process(params, stats, rgb, w, h)       # guetzli::Process(RGB)
"""
from .api import (Params, ProcessStats, process, process_image, process_jpeg, butteraugli_score_for_quality,
                  DeviceImage, load_library, library_path, write_jpeg, counters,
                  process_tiled_threads, process_tiled, dist_unique_id, dist_init, dist_shutdown,
                  last_error, Comparator, ComparatorSet, ButteraugliBatch, adaptive_quantization,
                  butteraugli_srgb, decode_jpeg)

__all__ = ["Params", "ProcessStats", "process", "process_image", "process_jpeg", "butteraugli_score_for_quality",
           "DeviceImage", "load_library", "library_path", "write_jpeg", "counters",
           "process_tiled_threads", "process_tiled", "dist_unique_id", "dist_init", "dist_shutdown", "last_error",
           "Comparator", "ComparatorSet", "ButteraugliBatch", "adaptive_quantization", "butteraugli_srgb",
           "decode_jpeg"]
