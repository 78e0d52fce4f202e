"""TEST INFRASTRUCTURE ONLY.  fp64, materialised restatement of the auxiliary loss of the reference's FSQRegularizer
(vidtok/modules/regularizers.py:200-204,228-245): the independent reference the device kernels (csrc/fsq_aux.cu) are
compared against.  The tokens x codebook distance and its softmax are formed explicitly, a bounded number of entries at
a time, so that production token counts fit in memory (on the CPU or on a GPU)."""
import torch
from torch import Tensor

from oracle.vidtok_oracle import fsq_regularize


def fsq_aux_parts(h: Tensor, levels, inv_temperature: float = 100.0, token_chunk_elems: int = 1 << 25):
    """The per-segment parts of FSQRegularizer's auxiliary loss (regularizers.py:228-242), fp64 and materialised: the
    tokens x codebook distance and its softmax are formed explicitly, `token_chunk_elems` entries at a time so that
    production token counts fit in memory.  h: the pre-bound encoder output [B,d,...] (any device).
    Returns (per_sample_entropy, avg_prob [J], commit_loss) as fp64 tensors (before the distributed mean)."""
    lv = torch.tensor(list(levels), dtype=torch.int64, device=h.device)
    basis = torch.cumprod(torch.tensor([1] + list(levels[:-1]), dtype=torch.int64, device=h.device), dim=0)
    J = int(torch.prod(lv))
    half_w = lv // 2
    j = torch.arange(J, device=h.device).unsqueeze(-1)
    codebook = (((j // basis) % lv) - half_w).double() / half_w.double()        # implicit_codebook, :114,180-198
    d = len(levels)
    z = h.detach().permute(0, *range(2, h.dim()), 1).reshape(-1, d)              # b d ... -> (b n) d
    n_tok = z.shape[0]
    zd = z.double()
    step = max(1, token_chunk_elems // J)
    ent = torch.zeros((), dtype=torch.float64, device=h.device)
    avg = torch.zeros(J, dtype=torch.float64, device=h.device)
    for a in range(0, n_tok, step):
        prob = (2.0 * inv_temperature * (zd[a:a + step] @ codebook.t())).softmax(dim=-1)   # softmax(-distance * inv_T)
        ent += (-prob * prob.clamp(min=1e-5).log()).sum()
        avg += prob.sum(dim=0)
        del prob
    codes = fsq_regularize(h.detach().float().cpu(), levels)[0].to(h.device)      # quantize(): bit-exact fp32 codes
    commit = ((h.detach().double() - codes.double()) ** 2).mean()
    return ent / n_tok, avg / n_tok, commit


def fsq_entropy_loss_weight(n_steps, entropy_loss_weight, annealing_steps, annealing_factor):
    """FSQRegularizer.calculate_entropy_loss_weight, regularizers.py:200-204."""
    if n_steps >= annealing_steps:
        return entropy_loss_weight
    start = annealing_factor * entropy_loss_weight
    return start - (n_steps / annealing_steps) * (start - entropy_loss_weight)


def fsq_aux_combine(per_sample_entropy, avg_prob, commit, entropy_loss_weight=0.1, entropy_loss_annealing_steps=2000,
                    entropy_loss_annealing_factor=3.0, commitment_loss_weight=0.25, diversity_gamma=1.0, n_steps=0):
    """regularizers.py:241-245,264-266 on the parts of one regularizer call (avg_prob after any distributed mean).
    Returns a dict of fp64 scalars: per_sample_entropy, codebook_entropy, commit_loss, aux_loss."""
    cbe = (-avg_prob * avg_prob.clamp(min=1e-5).log()).sum()
    w = fsq_entropy_loss_weight(n_steps, entropy_loss_weight, entropy_loss_annealing_steps, entropy_loss_annealing_factor)
    aux = (per_sample_entropy - diversity_gamma * cbe) * w + commit * commitment_loss_weight
    return {"per_sample_entropy": per_sample_entropy, "codebook_entropy": cbe, "commit_loss": commit, "aux_loss": aux}


def fsq_aux_loss(h: Tensor, levels, inv_temperature: float = 100.0, n_steps: int = 0, **weights):
    """reg_log['aux_loss'] of FSQRegularizer.forward (regularizers.py:232-245) in fp64, not distributed.  `weights`:
    entropy_loss_weight, entropy_loss_annealing_steps, entropy_loss_annealing_factor, commitment_loss_weight,
    diversity_gamma (defaults: the shipped FSQ configs).  Returns the dict of fsq_aux_combine."""
    pse, avg, commit = fsq_aux_parts(h, levels, inv_temperature)
    return fsq_aux_combine(pse, avg, commit, n_steps=n_steps, **weights)
