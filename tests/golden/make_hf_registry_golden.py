"""Generates tests/golden/hf_registry_golden.json from THE REFERENCE's own model registry: every hf/* entry of
marqo.s2_inference.model_registry._get_hf_properties() (model_registry.py:616-851), as the reference declares it.
tests/test_hf_registry.py checks marqo_b200.model_registry against this file, field for field.

    python tests/golden/make_hf_registry_golden.py
"""
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import _reference_import  # noqa: E402

_reference_import.install()
from marqo.s2_inference import model_registry  # noqa: E402

props = model_registry._get_hf_properties()
(HERE / "hf_registry_golden.json").write_text(json.dumps(props, indent=1, ensure_ascii=False, sort_keys=True) + "\n")
print(len(props), "hf/* entries")
