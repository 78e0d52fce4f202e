"""Import-path compatibility package: the reference's YAML configs name their classes by dotted path
(e.g. `target: vidtok.models.autoencoder.AutoencodingEngine`, configs/vidtok_kl_causal_488_4chn.yaml:3).
The modules of the tokenizer hot path (vidtok.models.autoencoder[_v1_1], vidtok.modules.model_3dcausal[_v1_1],
vidtok.modules.regularizers, vidtok.modules.util, vidtok.modules.losses) re-export the vidtok_b200 implementations.

Everything else of the reference's `vidtok` package (vidtok.data.*, vidtok.modules.lpips, ...) is NOT shadowed: the
reference ships `vidtok/` as a namespace package (no __init__.py), so when a reference checkout is importable
(VIDTOK_REFERENCE_ROOT, or any sys.path entry that holds the reference's vidtok/data/), its directories are appended to
this package's __path__ -- `from vidtok.data.vidtok import VidTokValDataset` (scripts/inference_evaluate.py:20) then
resolves to the reference's file while `vidtok.models.autoencoder` resolves to the CUDA path."""
import os as _os
import sys as _sys

_HERE = _os.path.dirname(_os.path.abspath(__file__))


def _reference_pkg_dir():
    cands = []
    env = _os.environ.get("VIDTOK_REFERENCE_ROOT")
    if env:
        cands.append(env)
    cands += [p or "." for p in _sys.path]
    for root in cands:
        d = _os.path.join(_os.path.abspath(root), "vidtok")
        if d != _HERE and _os.path.isdir(_os.path.join(d, "data")) and _os.path.isfile(_os.path.join(d, "modules", "util.py")):
            return d
    return None


REFERENCE_PACKAGE_DIR = _reference_pkg_dir()


def overlay(path, sub=""):
    """Append the reference's directory for (sub)package `sub` to `path` (a package __path__); ours stays first."""
    if REFERENCE_PACKAGE_DIR:
        d = _os.path.join(REFERENCE_PACKAGE_DIR, sub) if sub else REFERENCE_PACKAGE_DIR
        if _os.path.isdir(d) and d not in path:
            path.append(d)


overlay(__path__)

from vidtok_b200.compat_util import compute_psnr, get_obj_from_str, instantiate_from_config, print0  # noqa: F401,E402
