"""Host-side mirror of the reference's encoder seam (SURVEY §8 a1, a6, boundary B1).

`vectorise()` keeps the reference's signature, batching order, output type and error behaviour
(src/marqo/s2_inference/s2_inference.py:48-69, :123-158, :705-749); underneath, `model.encode()` is served by the
CUDA engine through the C ABI (`marqo_b200.loaders`).  Inside a real Marqo deployment the same loader classes are
registered into `MODEL_PROPERTIES['loaders']` (see INTEGRATION.md) and Marqo's own `vectorise` is used; this module
is the stand-alone equivalent for environments where `marqo` itself cannot be imported (SURVEY §0).

There is no CPU fallback: a `device` that is not `cuda[:N]` is rejected.
"""
from __future__ import annotations

import datetime
import os
import threading
from enum import Enum
from typing import Any, Dict, List, Optional, Sequence, Union

import numpy as np

from . import model_registry
from .inference_cache import MarqoInferenceCache
from .errors import (ConfigurationError, InternalError, InvalidModelPropertiesError, ModelCacheManagementError,
                     ModelLoadError, ModelNotInCacheError, UnknownModelError, VectoriseError)

try:  # optional at import time: PIL / torch are only needed for image and tensor content
    from PIL import UnidentifiedImageError
except Exception:  # pragma: no cover
    class UnidentifiedImageError(Exception):
        pass


class Modality(str, Enum):
    """src/marqo/s2_inference/multimodal_model_load.py:35-39"""
    TEXT = "language"
    IMAGE = "image"
    VIDEO = "video"
    AUDIO = "audio"


class AvailableModelsKey:
    """src/marqo/tensor_search/enums.py (AvailableModelsKey)"""
    model = "model"
    most_recently_used_time = "most_recently_used_time"
    model_size = "model_size"


# {"model_cache_key": {"model": obj, "most_recently_used_time": t, "model_size": gb}}  (s2_inference.py:37-41)
_available_models: Dict[str, Dict[str, Any]] = dict()
lock = threading.Lock()

DEFAULT_MAX_VECTORISE_BATCH_SIZE = 16  # src/marqo/api/configs.py:38 (MARQO_MAX_VECTORISE_BATCH_SIZE)


def get_default_normalization() -> bool:
    return True  # src/marqo/s2_inference/configs.py


def _get_max_vectorise_batch_size() -> int:
    """s2_inference.py:236-257: env var, must be an integer >= 1."""
    raw = os.environ.get("MARQO_MAX_VECTORISE_BATCH_SIZE", str(DEFAULT_MAX_VECTORISE_BATCH_SIZE))
    try:
        batch_size = int(raw)
    except (ValueError, TypeError) as e:
        raise ConfigurationError(f"Could not parse environment variable MARQO_MAX_VECTORISE_BATCH_SIZE={raw!r}. "
                                 f"Please make sure it is a positive integer") from e
    if batch_size < 1:
        raise ConfigurationError("MARQO_MAX_VECTORISE_BATCH_SIZE must be a positive integer")
    return batch_size


def generate_batches(seq: Sequence, batch_size: int):
    """src/marqo/tensor_search/utils.py:334-341"""
    if batch_size < 1:
        raise ValueError("Batch size must be greater than 0")
    for i in range(0, len(seq), batch_size):
        yield seq[i:i + batch_size]


def _create_model_cache_key(model_name: str, device: str, model_properties: dict = None) -> str:
    """s2_inference.py:260-283 — same key format (the eject-model API depends on it)."""
    if model_properties is None:
        model_properties = dict()
    return (model_name + "||" + model_properties.get('name', '') + "||" + str(model_properties.get('dimensions', ''))
            + "||" + model_properties.get('type', '') + "||" + str(model_properties.get('tokens', '')) + "||" + device)


def validate_model_properties(model_name: str, model_properties: Optional[dict]) -> dict:
    """s2_inference.py:340-407 reduced to the three loader types this engine serves: explicit properties must carry
    `dimensions` and a known `type`; otherwise the name is looked up in the registry."""
    if model_properties is None:
        return model_registry.get_model_properties(model_name)
    if not isinstance(model_properties, dict):
        raise InvalidModelPropertiesError("model_properties must be a dict")
    props = dict(model_properties)
    if "dimensions" not in props:
        raise InvalidModelPropertiesError(f"model_properties for {model_name} is missing the required key `dimensions`")
    mtype = props.get("type")
    alias = {"open_clip": model_registry.TYPE_OPEN_CLIP, "hf": model_registry.TYPE_HF,
             "hf_stella": model_registry.TYPE_HF_STELLA}
    props["type"] = alias.get(mtype, mtype)
    if props["type"] not in alias.values():
        raise InvalidModelPropertiesError(
            f"model type `{mtype}` is not served by the H100 engine (supported: open_clip, hf, hf_stella)")
    if "arch" not in props:
        base = model_registry.find_model(model_name)
        if base is None:
            served = model_registry.served_models()
            base = next((e for e in served.values() if e["name"] == props.get("name")), None)
        if base is None:
            raise InvalidModelPropertiesError(
                f"model_properties for {model_name} needs an `arch` block (or a registry name) to size the encoder")
        import copy
        props["arch"] = copy.deepcopy(base["arch"])
    if props["type"] in (model_registry.TYPE_HF, model_registry.TYPE_HF_STELLA):
        props.setdefault("tokens", 128)  # hugging_face_model_properties.py: default 128
    return props


def _validate_device(device: str) -> int:
    if not isinstance(device, str) or not device.startswith("cuda"):
        raise ModelLoadError(f"device={device!r}: the H100 engine only runs on CUDA devices (no CPU fallback)")
    if device == "cuda":
        return 0
    try:
        return int(device.split(":", 1)[1])
    except (IndexError, ValueError) as e:
        raise ModelLoadError(f"cannot parse device string {device!r}") from e


def _load_model(model_name: str, model_properties: dict, device: str, model_auth=None) -> Any:
    """s2_inference.py:520-568: loader = MODEL_PROPERTIES['loaders'][type]; loader(device=, model_properties=,
    model_auth=); model.load()."""
    from . import loaders
    loader = loaders.get_model_loader(model_properties.get("name"), model_properties)
    model = loader(device=device, model_properties=model_properties, model_auth=model_auth)
    model.load()
    return model


# Declared (not measured) model sizes in GB: src/marqo/s2_inference/constants.py:4-26; priorities
# model_properties["model_size"] > model name > model type > default (get_model_size, s2_inference.py:504-517)
MODEL_TYPE_SIZE_MAPPING = {"open_clip": 1, "clip": 1, "sbert": 0.7, "random": 0.1, "multilingual_clip": 5, "clip_onnx": 1,
                           "sbert_onnx": 0.7, "hf": 1}
MODEL_NAME_SIZE_MAPPING = {"vit-l-14": 1.5, "vit-g": 5, "vit-h": 5, "vit-bigg-14": 6}
DEFAULT_MODEL_SIZE = 0.66
DEFAULT_MAX_MODEL_MEMORY = 4   # GB per device, src/marqo/api/configs.py:35-36


def get_model_size(model_name: str, model_properties: dict):
    if "model_size" in model_properties:
        return model_properties["model_size"]
    name_info = (model_name + model_properties.get("name", "")).lower().replace("/", "-")
    for name, size in MODEL_NAME_SIZE_MAPPING.items():
        if name in name_info:
            return size
    return MODEL_TYPE_SIZE_MAPPING.get(_reference_type_name(model_properties.get("type", None)), DEFAULT_MODEL_SIZE)


def _reference_type_name(t):
    """this engine's loader types carry a b200_ prefix in the registry; sizes are declared per reference type"""
    return {model_registry.TYPE_OPEN_CLIP: "open_clip", model_registry.TYPE_HF: "hf",
            model_registry.TYPE_HF_STELLA: "hf_stella"}.get(t, t)


def _check_memory_threshold_for_model(device: str, model_size) -> bool:
    """s2_inference.py:460-501: sum of the DECLARED sizes of the models cached for this device + the new one must stay
    below MARQO_MAX_CUDA_MODEL_MEMORY / MARQO_MAX_CPU_MODEL_MEMORY; a model larger than the threshold is refused."""
    if device.startswith("cuda"):
        keys = [k for k in _available_models if k.endswith(device)]
        threshold = float(os.environ.get("MARQO_MAX_CUDA_MODEL_MEMORY", DEFAULT_MAX_MODEL_MEMORY))
    elif device.startswith("cpu"):
        keys = [k for k in _available_models if k.endswith("cpu")]
        threshold = float(os.environ.get("MARQO_MAX_CPU_MODEL_MEMORY", DEFAULT_MAX_MODEL_MEMORY))
    else:
        raise ModelCacheManagementError(f"Unable to check the device cache for device=`{device}`.")
    used_memory = sum(_available_models[k].get(AvailableModelsKey.model_size, DEFAULT_MODEL_SIZE) for k in keys)
    if model_size > threshold:
        raise ModelCacheManagementError(
            f"You are trying to load a model with size = `{model_size}` into device = `{device}`, which is larger than "
            f"the device threshold = `{threshold}`. Marqo CANNOT find enough space for the model. Please modify the "
            f"threshold by setting the environment variable `MARQO_MAX_CUDA_MODEL_MEMORY` or `MARQO_MAX_CPU_MODEL_MEMORY`.")
    return (used_memory + model_size) < threshold


def _validate_model_into_device(model_name: str, model_properties: dict, device: str) -> bool:
    """s2_inference.py:419-457: if the device's declared budget is exhausted, eject its models least-recently-used first
    until the new one fits (here `close()` frees the engine handle's memory; the reference relies on del + gc)."""
    model_size = get_model_size(model_name, model_properties)
    if _check_memory_threshold_for_model(device, model_size):
        return True
    on_device = sorted((k for k in list(_available_models) if k.endswith(device)),
                       key=lambda k: _available_models[k][AvailableModelsKey.most_recently_used_time])
    for key in on_device:
        entry = _available_models.pop(key)
        model = entry.get(AvailableModelsKey.model)
        if hasattr(model, "close"):
            model.close()
        if _check_memory_threshold_for_model(device, model_size):
            return True
    raise ModelCacheManagementError(
        f"Marqo CANNOT find enough space to load model = `{model_name}` in device = `{device}`.\n"
        f"Marqo tried to eject all the models on this device = `{device}` but still can't find enough space. \n"
        f"Please use a smaller model or increase the memory threshold.")


def _update_available_models(model_cache_key: str, model_name: str, validated_model_properties: dict, device: str,
                             normalize_embeddings: bool, model_auth=None) -> None:
    """s2_inference.py:286-337: load on first use under the module lock (after making room on the device), fail fast if
    another thread is loading."""
    if model_cache_key not in _available_models:
        model_size = get_model_size(model_name, validated_model_properties)
        if lock.locked():
            raise ModelCacheManagementError(
                "Request rejected, as this request attempted to update the model cache, while "
                "another request was updating the model cache at the same time. "
                "Please wait for 10 seconds and send the request again ")
        with lock:
            _validate_model_into_device(model_name, validated_model_properties, device)
            try:
                now = datetime.datetime.now()
                _available_models[model_cache_key] = {
                    AvailableModelsKey.model: _load_model(model_name, validated_model_properties, device=device,
                                                          model_auth=model_auth),
                    AvailableModelsKey.most_recently_used_time: now,
                    AvailableModelsKey.model_size: model_size,
                }
            except Exception as e:
                raise ModelLoadError(
                    f"Unable to load model={model_name} on device={device} with normalization={normalize_embeddings}. "
                    f"If you are trying to load a custom model, please check that "
                    f"model_properties={ {k: v for k, v in validated_model_properties.items() if k != 'weights'} } "
                    f"is correct and Marqo has access to the weights file. Original error: {e}") from e
    else:
        try:
            _available_models[model_cache_key][AvailableModelsKey.most_recently_used_time] = datetime.datetime.now()
        except KeyError as e:
            raise ModelNotInCacheError(
                f"Marqo cannot renew model {model_name} on device {device} with normalization={normalize_embeddings}. "
                f"Maybe another thread is updating the model cache at the same time."
                f"Please wait for 10 seconds and send the request again.\n") from e


def eject_model(model_name: str, device: str, model_properties: dict = None) -> None:
    key = _create_model_cache_key(model_name, device, validate_model_properties(model_name, model_properties))
    entry = _available_models.pop(key, None)
    if entry is None:
        raise ModelNotInCacheError(f"The model_name `{model_name}` device `{device}` is not cached or found")
    model = entry[AvailableModelsKey.model]
    if hasattr(model, "close"):
        model.close()  # releases the engine handle's device memory (the reference relies on del + empty_cache)


def clear_loaded_models() -> None:
    for entry in list(_available_models.values()):
        m = entry.get(AvailableModelsKey.model)
        if hasattr(m, "close"):
            m.close()
    _available_models.clear()


def is_preprocess_image_model(model_properties: dict = None) -> bool:
    """s2_inference.py:180-185 (constants.PREPROCESS_IMAGE_MODEL_LIST = CLIP-type models; here: the open_clip loader)."""
    return _reference_type_name((model_properties or {}).get("type")) in ("open_clip", "clip")


def load_multimodal_model_and_get_preprocessors(model_name: str, model_properties: Optional[dict] = None,
                                                device: Optional[str] = None, model_auth=None,
                                                normalize_embeddings: bool = get_default_normalization()):
    """s2_inference.py:193-235: what add_documents calls before downloading images — the loaded model plus the per-
    modality preprocessors its download threads apply (add_docs.py:129-134).  For this engine `model.preprocess` only
    decodes to uint8 HWC; resize / crop / normalise run on the GPU."""
    if not device:
        raise InternalError(message="vectorise (internal function) cannot be called without setting device!")
    model_properties = validate_model_properties(model_name, model_properties)
    model_cache_key = _create_model_cache_key(model_name, device, model_properties)
    _update_available_models(model_cache_key, model_name, model_properties, device, normalize_embeddings,
                             model_auth=model_auth)
    model = _available_models[model_cache_key][AvailableModelsKey.model]
    preprocessors = {
        "image": getattr(model, "preprocess", None) if is_preprocess_image_model(model_properties) else None,
        "video": None,
        "audio": None,
        "text": None,
    }
    return model, preprocessors


def _inference_cache_from_env() -> MarqoInferenceCache:
    """s2_inference.py:43-45; defaults: size 0 (disabled), LRU (tensor_search/configs.py)."""
    raw = os.environ.get("MARQO_INFERENCE_CACHE_SIZE", "0")
    try:
        size = int(raw)
    except ValueError:
        raise ConfigurationError(f"MARQO_INFERENCE_CACHE_SIZE must be an integer, got {raw!r}")
    return MarqoInferenceCache(cache_size=size, cache_type=os.environ.get("MARQO_INFERENCE_CACHE_TYPE", "LRU"))


_marqo_inference_cache = _inference_cache_from_env()


def vectorise(model_name: str, content, model_properties: dict = None, device: str = None,
              normalize_embeddings: bool = get_default_normalization(), model_auth=None, enable_cache: bool = False,
              modality: Modality = Modality.TEXT, **kwargs) -> List[List[float]]:
    """s2_inference.py:48-69"""
    if not device:
        raise InternalError(message="vectorise (internal function) cannot be called without setting device!")
    validated_model_properties = validate_model_properties(model_name, model_properties)
    model_cache_key = _create_model_cache_key(model_name, device, validated_model_properties)
    _update_available_models(model_cache_key, model_name, validated_model_properties, device, normalize_embeddings,
                             model_auth=model_auth)
    if _marqo_inference_cache.is_enabled() and enable_cache:
        return _vectorise_with_cache(model_cache_key, content, normalize_embeddings, modality, **kwargs)
    return _encode_without_cache(model_cache_key, content, normalize_embeddings, modality, **kwargs)


def _vectorise_with_cache(model_cache_key: str, content, normalize_embeddings: bool, modality: Modality, **kwargs):
    """s2_inference.py:72-119: only STRINGS are cached; a list call encodes its misses (and every non-string element)
    in one batch, stores the string results, and puts the hits back at their positions."""
    cache = _marqo_inference_cache
    if isinstance(content, str):
        hit = cache.get(model_cache_key, content)
        if hit is not None:
            return _convert_cached_embeddings_to_output(hit)
        vectorised = _encode_without_cache(model_cache_key, content, normalize_embeddings, modality, **kwargs)
        cache.set(model_cache_key, content, vectorised[0])
        return vectorised
    if not isinstance(content, list):
        raise TypeError(f"Unsupported content type: {type(content).__name__}")
    misses, hits = [], []
    for loc, item in enumerate(content):
        hit = cache.get(model_cache_key, item) if isinstance(item, str) else None
        if hit is None:
            misses.append(item)
        else:
            hits.append((loc, hit))
    if not misses:
        return [vector for _, vector in hits]
    outputs = _encode_without_cache(model_cache_key, misses, normalize_embeddings, modality, **kwargs)
    for item, vector in zip(misses, outputs):
        if isinstance(item, str):
            cache.set(model_cache_key, item, vector)
    for loc, vector in hits:          # ascending positions: each insert lands where the hit was in `content`
        outputs.insert(loc, vector)
    return outputs


def _convert_cached_embeddings_to_output(cached_embeddings: List[float]) -> List[List[float]]:
    """s2_inference.py:689-705"""
    if not isinstance(cached_embeddings, list):
        raise TypeError(f"expected a list of floats but received {type(cached_embeddings)}")
    if not isinstance(cached_embeddings[0], float):
        raise TypeError(f"expected a list of floats but received {type(cached_embeddings[0])}")
    return [cached_embeddings]


def _is_tensor(x) -> bool:
    return type(x).__module__.startswith("torch") and hasattr(x, "detach")


def _convert_tensor_to_numpy(output) -> np.ndarray:
    """s2_inference.py:677-686"""
    if _is_tensor(output):
        return output.to('cpu').detach().numpy()
    if isinstance(output, np.ndarray):
        return output
    raise ValueError(f"Marqo received an unexpected output type=`{type(output).__name__}`from encode function.")


def _encode_without_cache(model_cache_key: str, content, normalize_embeddings: bool, modality: Modality,
                          **kwargs) -> List[List[float]]:
    """s2_inference.py:123-158: str / tensor content goes to encode() whole; list content is cut into sub-batches of
    MARQO_MAX_VECTORISE_BATCH_SIZE, encoded in order and concatenated."""
    try:
        model = _available_models[model_cache_key][AvailableModelsKey.model]
        if isinstance(content, str):
            vectorised = model.encode(content, normalize=normalize_embeddings, modality=modality, **kwargs)
        elif _is_tensor(content):
            vectorised = model.encode(content, normalize=normalize_embeddings, modality=modality, **kwargs)
        else:
            vector_batches = []
            batch_size = _get_max_vectorise_batch_size()
            for batch in generate_batches(content, batch_size=batch_size):
                if modality is None:
                    modality = infer_modality(batch[0] if isinstance(batch[0], (str, bytes)) else batch)
                infer = kwargs.pop('infer', False if modality == Modality.TEXT else True)
                encoded_batch = model.encode(batch, modality=modality, normalize=normalize_embeddings, infer=infer,
                                             **kwargs)
                vector_batches.append(_convert_tensor_to_numpy(encoded_batch))
            if not vector_batches or all(len(batch) == 0 for batch in vector_batches):
                raise RuntimeError(f"Vectorise created an empty list of batches! Content: {content}")
            vectorised = np.concatenate(vector_batches, axis=0)
    except (UnidentifiedImageError, OSError) as e:
        if isinstance(e, UnidentifiedImageError) or "image file is truncated" in str(e):
            raise VectoriseError(f"Could not process given image: {content}. Original Error message: {e}") from e
        raise e
    return _convert_vectorized_output(vectorised)


def _check_output_type(output) -> bool:
    """s2_inference.py:622-648"""
    if not isinstance(output, list):
        return False
    elif len(output) == 0:
        raise ValueError("received empty input")
    if not isinstance(output[0], list):
        return False
    elif len(output[0]) == 0:
        raise ValueError("received empty input")
    if not isinstance(output[0][0], (float, int)):
        return False
    return True


def _convert_vectorized_output(output, fp16: bool = False) -> List[List[float]]:
    """s2_inference.py:705-749"""
    if _check_output_type(output):
        return output
    if _is_tensor(output):
        if output.ndim == 1:
            output = output.unsqueeze(0)
        output = output.detach().to("cpu").tolist()
    elif isinstance(output, np.ndarray):
        if output.ndim == 1:
            output = output[np.newaxis, :]
        output = output.tolist()
    elif isinstance(output, list):
        if _is_tensor(output[0]):
            output = [_o.detach().to("cpu").tolist() for _o in output]
        elif isinstance(output[0], np.ndarray):
            output = [_o.tolist() for _o in output]
        else:
            raise TypeError(f"unsupported nested list with elements of type {type(output[0])}")
    else:
        raise TypeError(f"unsupported output type of {type(output)}")
    if fp16:
        output = np.array(output).astype(np.float16).tolist()
    if _check_output_type(output):
        return output
    raise TypeError(f"unable to convert input of type {type(output)} to a list of lists of floats")


# --------------------------------------------------------------------------------------------- modality routing
_IMAGE_EXTS = {'.jpg', '.png', '.bmp', '.jpeg'}  # image_download.py:23-24


def _looks_like_url(s: str) -> bool:
    """Stand-in for validators.url (not installed here): scheme://host[...] with no whitespace."""
    import re
    return re.match(r"^[a-z][a-z0-9+.-]*://[^\s/$.?#][^\s]*$", s, re.IGNORECASE) is not None


def _is_image(inputs) -> bool:
    """src/marqo/core/inference/image_download.py:28-71 — decided by the FIRST element only."""
    if isinstance(inputs, list):
        if len(inputs) == 0:
            raise UnidentifiedImageError("received empty list, expected at least one element.")
        thing = inputs[0]
    else:
        thing = inputs
    if isinstance(thing, str):
        _, extension = os.path.splitext(thing.lower())
        if extension in _IMAGE_EXTS:
            return True
        if os.path.isfile(thing):
            raise UnidentifiedImageError(
                f"local file [{thing}] extension {extension} does not match allowed file types of {_IMAGE_EXTS}")
        return _looks_like_url(thing)
    if isinstance(thing, np.ndarray) or _is_tensor(thing) or type(thing).__module__.startswith("PIL."):
        return True
    if type(thing).__name__ == "EncodedImage":   # extension: a still-encoded image from this engine's own preprocessor
        return True                              # (marqo_b200/image_decode.py), decoded on the GPU by encode_image
    raise UnidentifiedImageError(f"expected type Image or str for inputs but received type {type(thing)}")


def infer_modality(content) -> Modality:
    """src/marqo/s2_inference/multimodal_model_load.py:148-200 without the network probe (no egress here): URLs are
    classified by extension only."""
    if isinstance(content, str):
        if not _looks_like_url(content):
            return Modality.TEXT
        extension = content.split('.')[-1].lower()
        if extension in ['jpg', 'jpeg', 'png', 'gif', 'webp']:
            return Modality.IMAGE
        elif extension in ['mp4', 'avi', 'mov']:
            return Modality.VIDEO
        elif extension in ['mp3', 'wav', 'ogg']:
            return Modality.AUDIO
        return Modality.TEXT
    return Modality.TEXT


# --------------------------------------------------------------------------------------------- fusion (a7)
def fuse_weighted_vectors(vectors: Sequence[Sequence[float]], weights: Sequence[float],
                          normalize: bool) -> List[float]:
    """Weighted-mean fusion + renormalise, arithmetic of src/marqo/tensor_search/tensor_search.py:1953-1973 (query
    side; skips the division when the norm is 0) — np.mean of the weighted vectors in fp64."""
    weighted_vectors = [np.asarray(vec) * weight for vec, weight in zip(vectors, weights)]
    merged_vector = np.mean(weighted_vectors, axis=0)
    if normalize:
        norm = np.linalg.norm(merged_vector, axis=-1, keepdims=True)
        if norm > 0:
            merged_vector /= np.linalg.norm(merged_vector, axis=-1, keepdims=True)
    return list(merged_vector)


def fuse_multimodal_field(embeddings: Sequence[Sequence[float]], weights: Sequence[float],
                          normalize: bool) -> List[float]:
    """Document-side multimodal combination, src/marqo/core/inference/tensor_fields_container.py:355-365."""
    combo_embeddings = [np.array(e) * w for e, w in zip(embeddings, weights)]
    vector_chunk = np.squeeze(np.mean(combo_embeddings, axis=0))
    if normalize:
        vector_chunk = vector_chunk / np.linalg.norm(vector_chunk)
    return vector_chunk.tolist()
