"""index-tts_b200 — H100-native (sm_90a) compute path behind the IndexTTS `.infer()` entry
points.  Host side: a ctypes shim over the C-ABI library `libidxtts.so` (include/idxtts.h) and
mirrors of the reference's operator interfaces (`gpt.UnifiedVoice.inference_speech`,
`bigvgan.BigVGAN.forward`, `s2mel` CFM).  PyTorch tensors are containers only."""
__version__ = "0.1.0"
