"""Local `from_pretrained` plumbing of the pipeline boundary (mirror of /root/reference/src/pyannote/audio/core/
pipeline.py:50-148 `expand_subfolders`, :153-334 `Pipeline.from_pretrained`, and pipelines/utils/getter.py `get_model` /
`get_plda`), without the Hugging Face hub: a community-1 style directory

    config.yaml                      pipeline: {name: pyannote.audio.pipelines.SpeakerDiarization,
    segmentation/pytorch_model.bin              params: {segmentation: $model/segmentation, embedding: $model/embedding,
    embedding/pytorch_model.bin                          plda: $model/plda, clustering: VBxClustering, ...}}
    plda/{xvec_transform,plda}.npz   params: {clustering: {threshold, Fa, Fb}, segmentation: {min_duration_off}}

is resolved entirely on the host (plain `yaml` + `torch.load`); hub identifiers are refused (no network here).
"""
from __future__ import annotations

import os
from pathlib import Path
from typing import Mapping, Optional, Tuple

CONFIG_NAME = "config.yaml"                                 # utils/hf_hub.py AssetFileName.Pipeline


def _expand_one(value: str, model_id, parent_subfolder, parent_revision, cache_dir, token) -> dict:
    subfolder = "/".join(value.split("/")[1:])
    if "@" in subfolder:                                    # "$model/sub@rev"
        subfolder, revision = subfolder.split("@")
    else:
        revision = parent_revision
    if parent_subfolder:
        subfolder = f"{parent_subfolder.rstrip('/')}/{subfolder.lstrip('/')}"
    return {"checkpoint": model_id, "revision": revision, "subfolder": subfolder, "token": token, "cache_dir": cache_dir}


def expand_subfolders(config, model_id=None, parent_subfolder: Optional[str] = None,
                      parent_revision: Optional[str] = None, cache_dir=None, token=None) -> None:
    """In place: every "$model/{subfolder}[@revision]" string of a (nested) dict / list becomes
    {"checkpoint": model_id, "revision", "subfolder", "token", "cache_dir"} (core/pipeline.py:50-148)."""
    if isinstance(config, dict):
        items = list(config.items())
    elif isinstance(config, list):
        items = list(enumerate(config))
    else:
        return
    for key, value in items:
        if isinstance(value, str) and value.startswith("$model/"):
            config[key] = _expand_one(value, model_id, parent_subfolder, parent_revision, cache_dir, token)
        else:
            expand_subfolders(value, model_id, parent_subfolder=parent_subfolder, parent_revision=parent_revision,
                              cache_dir=cache_dir, token=token)


def is_checkpoint_spec(value) -> bool:
    """What `get_model` / `get_plda` resolve: a path, or a mapping produced by expand_subfolders.  (State dicts are
    mappings too, but have no "checkpoint" entry; model / PLDA instances are passed through untouched.)"""
    if isinstance(value, (str, Path)):
        return True
    return isinstance(value, Mapping) and "checkpoint" in value


def _local(spec) -> Tuple[str, dict]:
    if isinstance(spec, (str, Path)):
        return str(spec), {}
    kw = {k: spec[k] for k in ("subfolder", "revision", "token", "cache_dir") if spec.get(k) is not None}
    return str(spec["checkpoint"]), kw


def get_model(model, token=None, cache_dir=None):
    """pipelines/utils/getter.py get_model: instance | path | {"checkpoint": ...} -> Model in eval mode."""
    from .models import Model

    if isinstance(model, Model):
        return model.eval()
    if not is_checkpoint_spec(model):
        raise TypeError(f"Unsupported type ({type(model)}) for loading model: expected `str`, `dict` or `Model`.")
    checkpoint, kw = _local(model)
    return Model.from_pretrained(checkpoint, **kw).eval()


def get_plda(plda, token=None, cache_dir=None):
    """pipelines/utils/getter.py get_plda: instance | directory | {"checkpoint": ...} -> PLDA."""
    from .clustering import PLDA

    if isinstance(plda, PLDA):
        return plda
    if not is_checkpoint_spec(plda):
        raise TypeError(f"Unsupported type ({type(plda)}) for loading PLDA: expected `str`, `dict` or `PLDA`.")
    checkpoint, kw = _local(plda)
    return PLDA.from_pretrained(checkpoint, **kw)


def _pipeline_class(name: str):
    short = name.rsplit(".", 1)[-1]
    if short == "SpeakerDiarization":
        from .pipeline import SpeakerDiarization

        return SpeakerDiarization
    if short == "VoiceActivityDetection":
        from .vad import VoiceActivityDetection

        return VoiceActivityDetection
    if short == "SpeakerEmbedding":
        from .speaker_verification import SpeakerEmbedding

        return SpeakerEmbedding
    if short == "MultiLabelSegmentation":
        from .multilabel import MultiLabelSegmentation

        return MultiLabelSegmentation
    raise NotImplementedError(f"pipeline '{name}' has no CUDA implementation here (SpeakerDiarization, "
                              f"VoiceActivityDetection, SpeakerEmbedding and MultiLabelSegmentation are available)")


def resolve_pipeline(checkpoint, revision: Optional[str] = None, subfolder: Optional[str] = None, token=None,
                     cache_dir=None):
    """Host half of Pipeline.from_pretrained (core/pipeline.py:153-277): -> (class, constructor params with
    "$model/..." entries expanded, hyper-parameters or None).  Same argument checks and messages as the reference."""
    import yaml

    if isinstance(checkpoint, dict):
        if revision is not None:
            raise ValueError("Revisions cannot be used with local checkpoints.")
        if subfolder is not None:
            raise ValueError("Subfolder cannot be used when checkpoint is a config dictionary. ")
        model_id, config = Path.cwd(), checkpoint
    elif os.path.isdir(checkpoint):
        if revision is not None:
            raise ValueError("Revisions cannot be used with local checkpoints.")
        model_id = Path(checkpoint)
        config_yml = model_id / subfolder / CONFIG_NAME if subfolder else model_id / CONFIG_NAME
    elif os.path.isfile(checkpoint):
        if revision is not None:
            raise ValueError("Revisions cannot be used with local checkpoints.")
        if subfolder is not None:
            raise ValueError("Subfolder cannot be used when checkpoint is a path to a config.yaml file. ")
        model_id, config_yml = Path(checkpoint).parent, checkpoint
    else:
        if "@" in str(checkpoint):
            raise ValueError("Revisions must be passed with `revision` keyword argument.")
        raise ValueError(f"'{checkpoint}' is not a local pipeline checkpoint; Hugging Face hub identifiers cannot be "
                         f"downloaded here (no network): pass the directory that holds config.yaml")
    if not isinstance(checkpoint, dict):
        with open(config_yml, "r") as fp:
            config = yaml.load(fp, Loader=yaml.SafeLoader)
    expand_subfolders(config, model_id, parent_subfolder=subfolder, parent_revision=revision, token=token,
                      cache_dir=cache_dir)
    klass = _pipeline_class(config["pipeline"]["name"])
    params = dict(config["pipeline"].get("params", {}) or {})
    params.setdefault("token", token)
    params.setdefault("cache_dir", cache_dir)
    return klass, params, config.get("params", None)


class Pipeline:
    """`Pipeline.from_pretrained(directory | config.yaml | config dict)` for local checkpoints."""

    @classmethod
    def from_pretrained(cls, checkpoint, revision: Optional[str] = None, hparams_file=None,
                        subfolder: Optional[str] = None, token=None, cache_dir=None, device=None):
        if hparams_file is not None:
            raise NotImplementedError("hparams_file (pyannote.pipeline optimisation output) is not supported")
        klass, params, hyper = resolve_pipeline(checkpoint, revision=revision, subfolder=subfolder, token=token,
                                                cache_dir=cache_dir)
        if cls is not Pipeline and not issubclass(klass, cls):
            raise ValueError(f"checkpoint describes a {klass.__name__}, not a {cls.__name__}")
        if device is not None:
            params["device"] = device
        pipeline = klass(**params)
        if hyper:
            pipeline.instantiate(hyper)
        return pipeline
