"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/fsq_aux/*.npz: the FSQ auxiliary loss (regularizers.py:232-245) of the
UNMODIFIED reference FSQRegularizer (the reference checkout, imported through oracle/ref_shim.py), next to the fp64 materialised oracle
(oracle/fsq_aux_oracle.py: fsq_aux_parts / fsq_aux_combine) and the deviation between the two.

Needs the reference checkout that oracle/ref_shim.py imports:   python oracle/make_golden_fsq_aux.py

Cases:
  (a) fix_<name>: the stored pre-bound latent `h` of every untiled FSQ fixture of tests/golden;
  (b) syn_<kind>_<levels>: seeded synthetic latents for 4, 5 and 6 digits and one odd level list -- peaked (|z| large),
      encoder-like and flat (z ~ 0, where the pruned entropy walk visits the most codes);
  (c) tiled_tiny_fsq_v11_tiled: the reference engine's tile_encode on that fixture's input and weights (aux_loss = mean over
      the chunks); every chunk's latent is stored;
  (d) dist2_<levels>: a two-rank gloo group on the CPU, spawned and joined here, each rank running the regularizer on its half
      of a synthetic batch (avg_prob all-reduced and divided by the world size).
The reference returns aux_loss only; its components come from the same unmodified class run with other weights:
  per_sample_entropy: entropy weight 1, gamma 0, commitment 0;  codebook_entropy: pse - (weight 1, gamma 1, commitment 0);
  commit_loss: entropy weight 0, commitment 1 (annealing off in all three).
"""
from __future__ import annotations

import json
import os
import sys
import tempfile
import warnings

warnings.filterwarnings("ignore")

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle.fsq_aux_oracle import fsq_aux_combine, fsq_aux_parts  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
OUT = os.environ.get("VIDTOK_GOLDEN_FSQ_AUX_OUT", os.path.join(GOLDEN, "fsq_aux"))
SHIPPED = dict(entropy_loss_weight=0.1, entropy_loss_annealing_steps=2000, entropy_loss_annealing_factor=3,
               commitment_loss_weight=0.25)
COMPONENTS = ("per_sample_entropy", "codebook_entropy", "commit_loss", "aux_loss")


def _reg(levels, **kw):
    from vidtok.modules.regularizers import FSQRegularizer
    return FSQRegularizer(list(levels), **kw)


def reference_components(h, levels):
    """fp32 values of the unmodified reference for one regularizer call (see the module docstring)."""
    def aux(**kw):
        with torch.no_grad():
            return float(_reg(levels, **kw)(h)[1]["aux_loss"])
    pse = aux(entropy_loss_weight=1.0, diversity_gamma=0.0)
    ent = aux(entropy_loss_weight=1.0, diversity_gamma=1.0)
    commit = aux(entropy_loss_weight=0.0, commitment_loss_weight=1.0)
    return {"per_sample_entropy": pse, "codebook_entropy": pse - ent, "commit_loss": commit, "aux_loss": aux(**SHIPPED)}


def oracle_components(h, levels):
    pse, avg, commit = fsq_aux_parts(h, levels)
    return {k: float(v) for k, v in fsq_aux_combine(pse, avg, commit, **SHIPPED).items()}


def deviation(ref, ora):
    return {k: abs(ref[k] - ora[k]) / max(abs(ora[k]), 1e-12) for k in COMPONENTS}


def save(name, arrays, meta):
    os.makedirs(OUT, exist_ok=True)
    arrays = dict(arrays)
    arrays["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **arrays)
    print(f"[fsq_aux] {name}: aux ref {meta['reference']['aux_loss']:.9g} oracle {meta['oracle']['aux_loss']:.9g} "
          f"max dev {max(meta['deviation'].values()):.3e}", flush=True)


def single(name, h, levels, source):
    ref, ora = reference_components(h, levels), oracle_components(h, levels)
    save(name, {"h": h.numpy()}, {"case": name, "kind": "single", "levels": list(levels), "source": source, "weights": SHIPPED,
                                  "reference": ref, "oracle": ora, "deviation": deviation(ref, ora), "torch": torch.__version__})


def synthetic(kind, levels, shape, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(shape, generator=g)
    scale = {"peaked": 2.5, "encoder": 0.5, "flat": 2e-3}[kind]
    return (z * scale).contiguous()


def tiled_case():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from make_golden import CASES, model_yaml
    from vidtok_b200.synth import synth_clip, synth_state_dict
    name = "tiny_fsq_v11_tiled"
    ykw, (B, T, H, W), chunk, _ = CASES[name]
    my = model_yaml(**ykw)
    ref = ref_shim.build_reference_model(my)
    shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items() if k.startswith(("encoder.", "decoder."))}
    ref.load_state_dict(synth_state_dict(shapes, seed=0), strict=False)
    ref.use_tiling, ref.t_chunk_enc = True, chunk
    x = synth_clip(B, T, H, W, seed=1234)
    seen = []
    hook = ref.regularization.register_forward_pre_hook(lambda mod, args: seen.append(args[0].detach().clone()))
    with torch.no_grad():
        _, log = ref.encode(x, return_reg_log=True)
    hook.remove()
    levels = list(my["params"]["regularizer_config"]["params"]["levels"])
    per_chunk = [oracle_components(hc, levels) for hc in seen]
    ora = {k: float(np.mean([c[k] for c in per_chunk])) for k in COMPONENTS}
    refc = {"aux_loss": float(log["aux_loss"])}
    arrays = {f"h{i}": hc.numpy() for i, hc in enumerate(seen)}
    save("tiled_" + name, arrays, {"case": "tiled_" + name, "kind": "tiled", "levels": levels, "source": name, "weights": SHIPPED,
                                   "n_chunks": len(seen), "reference": refc, "oracle": ora, "oracle_chunks": per_chunk,
                                   "deviation": {"aux_loss": abs(refc["aux_loss"] - ora["aux_loss"]) / abs(ora["aux_loss"])},
                                   "torch": torch.__version__})


def _rank(rank, world, init, levels, h_path, out_path):
    import torch.distributed as dist
    ref_shim.import_reference()
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    h = torch.from_numpy(np.load(h_path))
    half = h.shape[0] // world
    comps = reference_components(h[rank * half:(rank + 1) * half].contiguous(), levels)
    dist.destroy_process_group()
    with open(out_path + f".{rank}", "w") as f:
        json.dump(comps, f)


def dist_case(levels, seed):
    import torch.multiprocessing as mp
    h = synthetic("encoder", levels, (4, len(levels), 2, 8, 8), seed)
    with tempfile.TemporaryDirectory() as td:
        hp, out = os.path.join(td, "h.npy"), os.path.join(td, "out")
        np.save(hp, h.numpy())
        init = "file://" + os.path.join(td, "rendezvous")
        mp.start_processes(_rank, args=(2, init, list(levels), hp, out), nprocs=2, join=True, start_method="spawn")
        ranks = []
        for r in range(2):
            with open(out + f".{r}") as f:
                ranks.append(json.load(f))
    parts = [fsq_aux_parts(h[r * 2:(r + 1) * 2], levels) for r in range(2)]
    avg = (parts[0][1] + parts[1][1]) / 2
    ora = [{k: float(v) for k, v in fsq_aux_combine(p[0], avg, p[2], **SHIPPED).items()} for p in parts]
    name = "dist2_" + "".join(str(l) for l in levels)
    dev = [deviation(ranks[r], ora[r]) for r in range(2)]
    save(name, {"h": h.numpy()}, {"case": name, "kind": "dist2", "levels": list(levels), "world_size": 2, "weights": SHIPPED,
                                  "reference": ranks[0], "oracle": ora[0], "reference_ranks": ranks, "oracle_ranks": ora,
                                  "deviation": {k: max(d[k] for d in dev) for k in COMPONENTS}, "torch": torch.__version__})


def main():
    torch.set_num_threads(os.cpu_count())
    ref_shim.import_reference()
    for name in ("tiny_fsq_v10", "mid_fsq_v10", "tiny_fsq_nc", "tiny_fsq_888_v11", "cfg1_fsq_488_32768"):
        d = np.load(os.path.join(GOLDEN, name + ".npz"))
        meta = json.loads(bytes(d["meta_json"]).decode())
        levels = meta["model"]["params"]["regularizer_config"]["params"]["levels"]
        single("fix_" + name, torch.from_numpy(d["h"]), levels, name)
    synth = [((8, 8, 8, 8), (2, 4, 2, 16, 16)), ((8, 8, 8, 8, 8), (2, 5, 2, 8, 16)), ((8, 8, 8, 8, 8, 8), (1, 6, 1, 8, 16)),
             ((7, 5, 5, 5), (2, 4, 2, 16, 16))]
    for seed, (levels, shape) in enumerate(synth):
        for kind in ("peaked", "encoder", "flat"):
            single(f"syn_{kind}_" + "".join(str(l) for l in levels), synthetic(kind, levels, shape, 100 + seed), levels,
                   f"synthetic {kind} {list(shape)} seed {100 + seed}")
    tiled_case()
    dist_case((8, 8, 8, 8, 8), 7)


if __name__ == "__main__":
    main()
