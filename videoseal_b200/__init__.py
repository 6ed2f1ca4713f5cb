"""videoseal_b200: H100-native (sm_90a) implementation of VideoSeal's embed/detect hot path behind the
reference's `videoseal.load() / model.embed() / model.detect()` API (videoseal/__init__.py:13-17)."""

__version__ = "0.1"


def load(*args, **kwargs):
    """Same contract as `videoseal.load(card_name_or_Path)` (utils/cfg.py:181)."""
    from .cfg import setup_model_from_model_card
    return setup_model_from_model_card(*args, **kwargs)
