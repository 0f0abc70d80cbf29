"""masr_b200 — a H100-native (sm_90a) implementation of MASR's inference hot path
(fbank -> Conformer-family encoder -> CTC greedy / prefix beam) behind the reference's
``MASRPredictor.predict / predict_stream`` interface.  See DESIGN.md."""

__version__ = "0.1.0"

SUPPORT_MODEL = ['squeezeformer', 'efficient_conformer', 'conformer', 'deepspeech2']  # masr/__init__.py
