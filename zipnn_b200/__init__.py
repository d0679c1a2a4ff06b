"""zipnn_b200 -- the ZipNN encode/decode hot path on H100 (sm_90a).

Drop-in for the reference package surface that sits on the hot path
(reference zipnn/__init__.py:1):  `ZipNN`, `zipnn_safetensors`, `zipnn_hf` (the transformers
plugin for `.znn` checkpoints, zipnn/zipnn.py:1221-1565; see hf.py for how it differs).
"""
from .zipnn import DecodePipe, ZipNN
from .safetensors_io import (SafeOpen, compress_safetensors_file, decompress_safetensors_file,
                             decompress_safetensors_tensor, load_file, zipnn_safetensors)


from .hf import zipnn_hf


__all__ = ["ZipNN", "zipnn_safetensors", "SafeOpen", "compress_safetensors_file",
           "decompress_safetensors_file", "decompress_safetensors_tensor", "load_file", "DecodePipe", "zipnn_hf"]
