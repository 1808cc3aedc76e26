"""luminoth_b200: H100-native (sm_90a) inference engine for the Faster R-CNN /
SSD predict path of tryolabs/luminoth, behind Luminoth's own
PredictorNetwork / config-YAML surface.  No CPU fallback."""
from .config import get_config, default_config, override_config_params, set_prediction_filters  # noqa: F401

__version__ = '0.1'


def get_predictor(config, min_prob=None, max_detections=None, **kwargs):
    """``PredictorNetwork(config)`` after the caller-side config mutations of ``predict.py:246-259`` (pass
    ``min_prob=0.5, max_detections=100`` for the ``lumi predict`` defaults)."""
    from .predicting import PredictorNetwork
    return PredictorNetwork(set_prediction_filters(config, min_prob, max_detections), **kwargs)
