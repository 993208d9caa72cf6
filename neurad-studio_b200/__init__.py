"""neurad-studio_b200 -- H100-native (sm_90a) backend for NeuRAD's volumetric-rendering hot path.

Import as ``neurad_studio_b200`` (the top-level ``neurad_studio_b200.py`` shim maps the importable name onto
this directory, whose on-disk name carries a hyphen).
"""
from .config import (HashGridSettings, NeuRADConfig, NeuRADHashEncodingConfig, PRESETS, SamplingSettings, preset,  # noqa: F401
                     small_config)

__version__ = "0.1.0"
