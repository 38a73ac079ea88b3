"""ptlflow_b200 -- H100-native (sm_90a) backend for ptlflow's RAFT-family inference hot path.

Public surface mirrors ptlflow/__init__.py:65-285 for the models this backend covers:
``get_model``, ``get_model_reference``, ``get_model_names``, ``get_trainable_model_names``,
``load_checkpoint``, ``restore_model``.  Everything numerical on the hot path lives in
libptlflow_b200.so (include/ptlflow_b200.h); see DESIGN.md.
"""
from __future__ import annotations

from argparse import Namespace
from pathlib import Path
from typing import Any, Dict, List, Optional

import torch

from . import models  # noqa: F401  (registers the model classes)
from .utils.registry import _models_dict, _ptlflow_trained_models, _trainable_models

__version__ = "0.1.0"


def get_model_reference(model_name: str):
    """Return the class registered under ``model_name`` (ptlflow/__init__.py:128-159)."""
    try:
        return _models_dict[model_name]
    except KeyError:
        raise ValueError(f"Unknown model name: {model_name}. Choose from [{', '.join(sorted(_models_dict))}]") from None


def get_model_names() -> List[str]:
    return sorted(_models_dict.keys())


def get_trainable_model_names() -> List[str]:
    return sorted(set(_trainable_models))


def get_ptlflow_trained_model_names() -> List[str]:
    return sorted(set(_ptlflow_trained_models))


def _model_kwargs(args: Optional[Any]) -> Dict[str, Any]:
    """Constructor kwargs from ``args.model`` (a Namespace or dict; jsonargparse's ``init_args``
    nesting is accepted too), as the reference builds them in ptlflow/__init__.py:105-113."""
    if args is None:
        return {}
    m = getattr(args, "model", None) if not isinstance(args, dict) else args.get("model")
    if m is None:
        return {}
    if isinstance(m, Namespace):
        m = vars(m)
    m = dict(m)
    if "init_args" in m:
        inner = m["init_args"]
        m = dict(vars(inner) if isinstance(inner, Namespace) else inner)
    m.pop("class_path", None)
    return m


def get_model(model_name: str, ckpt_path: Optional[str] = None, args: Optional[Namespace] = None):
    """Instance of ``model_name`` configured by ``args.model.<kw>``, optionally restored from a
    checkpoint (ptlflow/__init__.py:65-125)."""
    model_ref = get_model_reference(model_name)
    model = model_ref(**_model_kwargs(args))
    if ckpt_path is None and args is not None and getattr(args, "ckpt_path", None) is not None:
        ckpt_path = args.ckpt_path
    return restore_model(model, ckpt_path)


def load_checkpoint(ckpt_path: str, model_ref) -> Dict[str, Any]:
    """Local file, or the name of one of ``model_ref.pretrained_checkpoints`` (downloaded through
    torch.hub's cache -- needs network on first use).  ptlflow/__init__.py:201-251."""
    if Path(ckpt_path).exists():
        return torch.load(ckpt_path, map_location="cpu", weights_only=True)
    table = getattr(model_ref, "pretrained_checkpoints", None)
    if not table:
        raise ValueError(f"Cannot find checkpoint {ckpt_path} for model {model_ref.__name__}")
    if ckpt_path not in table:
        raise ValueError(f"Invalid checkpoint name {ckpt_path}. Choose one from {{{','.join(table.keys())}}}")
    cache_dir = Path(torch.hub.get_dir()) / "checkpoints"
    return torch.hub.load_state_dict_from_url(table[ckpt_path], model_dir=str(cache_dir), map_location="cpu", check_hash=True, weights_only=True)


def restore_model(model, ckpt_path: Optional[str]):
    """Strict ``load_state_dict`` of ``ckpt['state_dict']`` + train_size / extra_params hparams
    (ptlflow/__init__.py:254-285)."""
    if ckpt_path is None:
        return model
    ckpt = load_checkpoint(ckpt_path, model.__class__)
    hp = ckpt.get("hyper_parameters", {})
    if "train_size" in hp:
        model.train_size = hp["train_size"]
    if "train_avg_length" in hp:
        model.train_avg_length = hp["train_avg_length"]
    for name, value in (hp.get("extra_params") or {}).items():
        model.add_extra_param(name, value)
    model.load_state_dict(ckpt["state_dict"])
    return model
