"""`indextts_b200.infer_v2_5.IndexTTS2` — the reference's entry-point class with its compute seams on the CUDA engine.

Same constructor and `.infer()` / `.infer_generator()` signatures as `indextts.infer_v2_5.IndexTTS2`
(infer_v2_5.py:77-80, 506-509, 570-573): the class builds the REFERENCE object with the reference's own config and
checkpoint loaders (so every loader quirk stays the reference's), then `dropin.attach()` rebinds the module-level seams
(merge_emovec, inference_speech, codec decode, length regulator, CFM, BigVGAN) to libidxtts.so.  Everything else of
`.infer()` — text front-end, prompt caching, segment loop, timing prints, file output — is the reference's code, unmodified.

The reference package must be importable (`pip install -e` of the index-tts checkout, or IDX_REFERENCE_ROOT pointing at
it); this module does not vendor it.  There is no PyTorch-compute fallback: without an H100 the constructor raises."""
import importlib
import os
import sys

from .dropin import attach


def _reference(module):
    root = os.environ.get("IDX_REFERENCE_ROOT")
    if root and root not in sys.path:
        sys.path.insert(0, root)
    try:
        return importlib.import_module(module)
    except ImportError as ex:  # pragma: no cover
        raise ImportError(f"{module} is not importable ({ex}); install the index-tts checkout or set IDX_REFERENCE_ROOT") from ex


class IndexTTS2:
    def __init__(self, cfg_path="checkpoints/config.yaml", model_dir="checkpoints", use_bf16=False, device=None,
                 use_cuda_kernel=None, use_deepspeed=False, use_accel=False, use_torch_compile=False, use_qwen_emo=False,
                 engine_device=0):
        ref = _reference("indextts.infer_v2_5")
        # use_cuda_kernel / use_accel / use_torch_compile / use_deepspeed select reference-side accelerations of the very
        # modules that are rebound below: they are forced off so the reference builds its plain modules (their weights
        # are what the engine loads) and nothing is compiled twice
        self._ref = ref.IndexTTS2(cfg_path=cfg_path, model_dir=model_dir, use_bf16=use_bf16, device=device, use_cuda_kernel=False,
                                  use_deepspeed=False, use_accel=False, use_torch_compile=False, use_qwen_emo=use_qwen_emo)
        attach(self._ref, device=engine_device)

    def infer(self, spk_audio_prompt, text, output_path, lang, emo_audio_prompt=None, emo_alpha=1.0, emo_vector=None,
              use_emo_text=False, emo_text=None, use_random=False, interval_silence=200, verbose=False,
              max_text_tokens_per_segment=120, stream_return=False, more_segment_before=0, duration_factor=1.0,
              text_normalization=True, **generation_kwargs):
        return self._ref.infer(spk_audio_prompt, text, output_path, lang, emo_audio_prompt=emo_audio_prompt, emo_alpha=emo_alpha,
                               emo_vector=emo_vector, use_emo_text=use_emo_text, emo_text=emo_text, use_random=use_random,
                               interval_silence=interval_silence, verbose=verbose,
                               max_text_tokens_per_segment=max_text_tokens_per_segment, stream_return=stream_return,
                               more_segment_before=more_segment_before, duration_factor=duration_factor,
                               text_normalization=text_normalization, **generation_kwargs)

    def infer_generator(self, *args, **kwargs):
        return self._ref.infer_generator(*args, **kwargs)

    def __getattr__(self, name):          # everything else (tokenizer, caches, gr_progress, ...) is the reference object's
        return getattr(self.__dict__["_ref"], name)
