"""pantomatrix_b200: H100-native (sm_90a) implementation of PantoMatrix's EMAGE audio->motion
inference hot path behind the reference's `models.emage_audio` module API."""
__version__ = "0.1.0"
