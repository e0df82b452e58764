"""facodec_b200 -- H100-native FAcodec encode -> quantize -> decode hot path (sm_90a CUDA
behind the reference's model.encoder / model.quantizer / model.decoder call surface)."""
from .modules import (Activation1d, CNNLSTM, Codec, CodecDecodePool, CodecStream, CodecStreamPool, Decoder, Encoder, Engine, FApredictors, FAquantizer, JDCNet, Munch,  # noqa: F401
                      Redecoder, ResamplePool, ResidualVQ, SessionState, VoiceConversionPool, VoiceConversionStream, VoiceConverter, build_model, f0_targets,
                      load_F0_models, log_norm, resample, resample_length, resample_table)
from ._lib import FacError  # noqa: F401

__all__ = ["build_model", "Encoder", "FAquantizer", "Decoder", "Redecoder", "Codec", "CodecStream", "CodecStreamPool", "CodecDecodePool", "VoiceConverter",
           "VoiceConversionStream", "VoiceConversionPool", "ResamplePool", "SessionState", "resample", "resample_length", "resample_table", "ResidualVQ", "Activation1d", "CNNLSTM", "FApredictors", "JDCNet", "load_F0_models", "f0_targets", "log_norm", "Engine", "Munch", "FacError"]
