"""`indextts_b200.infer.IndexTTS` — the v1 / v1.5 entry point (indextts/infer.py:29-32, 520-521) with its compute seams on
the CUDA engine: the reference object is built by the reference's own constructor, `dropin.attach_v1()` rebinds
`gpt.inference_speech`, the latent pass `gpt(..., return_latent=True)` and `bigvgan(latent, mel_ref)`; `.infer()` /
`.infer_fast()` stay the reference's code.  See infer_v2_5.py in this package for the import contract."""
from .dropin import attach_v1
from .infer_v2_5 import _reference


class IndexTTS:
    def __init__(self, cfg_path="checkpoints/config.yaml", model_dir="checkpoints", use_fp16=True, device=None,
                 use_cuda_kernel=None, engine_device=0):
        ref = _reference("indextts.infer")
        # the engine keeps the v1 GPT in fp32 (the reference's CPU configuration, BASELINE config 1); use_fp16 only
        # affects reference-side modules that are not on the rebound path
        self._ref = ref.IndexTTS(cfg_path=cfg_path, model_dir=model_dir, use_fp16=False, device=device, use_cuda_kernel=False)
        attach_v1(self._ref, device=engine_device)

    def infer(self, audio_prompt, text, output_path, verbose=False, max_text_tokens_per_segment=120, **generation_kwargs):
        return self._ref.infer(audio_prompt, text, output_path, verbose=verbose,
                               max_text_tokens_per_segment=max_text_tokens_per_segment, **generation_kwargs)

    def infer_fast(self, *args, **kwargs):
        return self._ref.infer_fast(*args, **kwargs)

    def __getattr__(self, name):
        return getattr(self.__dict__["_ref"], name)
