"""Generates tests/golden/multilingual_clip_golden.json from THE REFERENCE's own registry of M-CLIP models: every entry
of marqo.s2_inference.clip_utils.get_multilingual_clip_properties() (clip_utils.py:599-640) as the reference declares
it, with the size get_model_size (s2_inference.py:504-517, constants.py:6-25) declares for it under "model_size".
tests/test_multilingual_clip.py checks marqo_b200.model_registry and marqo_b200.s2_inference.get_model_size against
this file.

    python tests/golden/make_multilingual_clip_golden.py
"""
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import _reference_import  # noqa: E402

_reference_import.install()
import torchaudio  # noqa: E402

# the reference's languagebind package, which s2_inference imports, calls a torchaudio function removed since; it is
# never used by get_model_size
if not hasattr(torchaudio, "set_audio_backend"):
    torchaudio.set_audio_backend = lambda backend: None
from marqo.s2_inference import clip_utils, s2_inference  # noqa: E402

entries = clip_utils.get_multilingual_clip_properties()
golden = {name: {"properties": props, "model_size": s2_inference.get_model_size(name, props)}
          for name, props in entries.items()}
(HERE / "multilingual_clip_golden.json").write_text(json.dumps(golden, indent=1, ensure_ascii=False, sort_keys=True)
                                                    + "\n")
print(len(golden), "multilingual_clip entries")
