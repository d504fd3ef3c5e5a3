"""mlx-audio-swift_b200: H100-native (sm_90a) speech-inference hot path behind MLXAudio's protocols.

Everything numeric runs in `lib/libb200audio.so` (hand-written CUDA, C ABI in include/b200audio.h);
this package is the host-side mirror of the reference interface for that path.  No CPU fallback."""
from . import _ffi
from ._ffi import AudioGenerationError
from .dsp import (IncrementalMelSpectrogram, LogMel, compute_mel_spectrogram, hamming_window, hanning_window, mel_filters, power_to_db,
                  whisper_encoder_features)
from .snac import SNAC
from .llama_tts import AudioGenerationInfo, GenerateParameters, LlamaTTSModel
from .vyvo_tts import Qwen3Model
from .soprano_tts import SopranoModel
from .vocos import Vocos
from .encodec import Encodec, EncodecConfig, EncodecEncodedAudio
from .mimi import Mimi, MimiStreamingDecoder
from .loading import Weights, llama_config_from_json
from .whisper import STTGenerateParameters, STTOutput, StreamingConfig, StreamingInferenceSession, StreamingUpdate, WhisperModel
from .qwen3_tts import (Qwen3CodePredictorConfig, Qwen3GenerateParameters, Qwen3SpeakerEncoderConfig, Qwen3TalkerConfig, Qwen3TTSModel,
                        Qwen3TTSSpeakerEncoder, Qwen3TTSTalker)

__all__ = ["AudioGenerationError", "IncrementalMelSpectrogram", "LogMel", "compute_mel_spectrogram", "hanning_window", "hamming_window", "power_to_db",
           "mel_filters", "whisper_encoder_features", "SNAC", "LlamaTTSModel", "Qwen3Model", "SopranoModel", "GenerateParameters",
           "AudioGenerationInfo", "Vocos", "Weights", "llama_config_from_json", "Encodec", "EncodecConfig", "EncodecEncodedAudio", "Mimi", "MimiStreamingDecoder", "WhisperModel", "STTGenerateParameters", "STTOutput",
           "StreamingInferenceSession", "StreamingConfig", "StreamingUpdate",
           "Qwen3TTSTalker", "Qwen3TTSModel", "Qwen3TalkerConfig", "Qwen3CodePredictorConfig", "Qwen3GenerateParameters",
           "Qwen3TTSSpeakerEncoder", "Qwen3SpeakerEncoderConfig"]


def device_count() -> int:
    return int(_ffi.lib().b2a_device_count())


def launch_count() -> int:
    return int(_ffi.lib().b2a_launch_count())
