"""State-dict key mapping between ``NequIPEnergyModel`` and the reference's ``NequIPGNNEnergyModel``.

The reference assembles a ``SequentialGraphNetwork`` with the module names of
nequip/model/nequip_models.py:288-399 -- ``type_embed`` (``NodeTypeEmbed.embed_module``, nn/embedding/node.py:75),
``layer{i}_convnet.conv.{linear_1, linear_2, sc, edge_mlp.mlp.{2k}}`` (nn/convnetlayer.py:142,
nn/interaction_block.py:82-146, nn/mlp.py:134-192), ``per_atom_energy_readout.mlp_module`` (nn/mlp.py:62),
``per_type_energy_scale_shift.{scales, shifts}`` (nn/atomwise.py:206-233), in a model with a pair potential
``pair_potential.{atomic_numbers, _qqr2exesquare}`` (model/energy_modules.py:20-27, nn/pair_potential.py:336-358), and
``edge_norm._rmax_recip`` (nn/embedding/_edge.py:47-53: ``1 / r_max`` or the [T * T] per-edge-type table) --
wrapped in ``ForceStressOutput.func`` and possibly ``GraphModel.model``.  Parameters are matched by SUFFIX, so any
wrapper prefix is accepted; e3nn's persistent buffers (``tp_scatter.tp.*``, ``*.output_mask``, ...) carry no
learnable state and are ignored.

Flattening conventions assumed for the e3nn weights (SURVEY.md Appendix A.4; e3nn itself is not installed here, so
this is stated, not verified): ``o3.Linear.weight`` = concatenation over instructions (i_in-major over equal irreps)
of row-major ``[mul_in, mul_out]`` blocks; ``FullyConnectedTensorProduct.weight`` = concatenation of ``[mul_in,
num_attr, mul_out]`` blocks; ``ScalarLinearLayer.weight`` = ``[in, out]``.
"""
from __future__ import annotations

import re
from typing import Dict, Tuple

import torch

_IGNORED = re.compile(r"(tp_scatter\.tp\.|\.output_mask$|_w3j|\.tp\._|norm_const$|\.alpha$|bessel_weights$|_empty$)")


RMAX_RECIP_KEY = "edge_norm._rmax_recip"


def reference_key_map(num_layers: int, radial_mlp_depth: int = 1, pair_potential: bool = False,
                      per_edge_type_cutoff: bool = False) -> Dict[str, str]:
    """reference key suffix -> ``NequIPEnergyModel.state_dict()`` key (``pair_potential``: the model has ZBL;
    ``per_edge_type_cutoff``: the model has per-edge-type cutoffs, buffer ``rmax_recip``)."""
    m = {
        "type_embed.embed_module.weight": "type_embed.weight",
        "per_atom_energy_readout.mlp_module.mlp.0.weight": "readout.mlp.0.weight",
        "per_type_energy_scale_shift.scales": "scales",
        "per_type_energy_scale_shift.shifts": "shifts",
    }
    for i in range(num_layers):
        ref, ours = f"layer{i}_convnet.conv.", f"layers.{i}.conv."
        m[ref + "linear_1.weight"] = ours + "linear_1.weight"
        m[ref + "linear_2.weight"] = ours + "linear_2.weight"
        if i != 0:
            m[ref + "sc.weight"] = ours + "sc.weight"
        for q in range(radial_mlp_depth + 1):
            m[ref + f"edge_mlp.mlp.{2 * q}.weight"] = ours + f"edge_mlp.mlp.{2 * q}.weight"
    if pair_potential:
        for k in ("pair_potential.atomic_numbers", "pair_potential._qqr2exesquare"):
            m[k] = k
    if per_edge_type_cutoff:
        m[RMAX_RECIP_KEY] = "rmax_recip"
    return m


def _key_map(model) -> Dict[str, str]:
    cfg = model.config
    return reference_key_map(cfg["num_layers"], cfg["radial_mlp_depth"], cfg.get("pair_potential") is not None,
                             cfg.get("per_edge_type_cutoff") is not None)


def _check_rmax_recip(model, v: torch.Tensor, rk: str) -> None:
    """The checkpoint's ``edge_norm._rmax_recip`` must be what the model computes with: its own [T * T] table, or
    ``1 / r_max`` (a scalar, or a table of it) for a model built without ``per_edge_type_cutoff``."""
    T = len(model.config["type_names"])
    if model.per_edge_type_cutoff is not None:
        want = model.rmax_recip.detach().cpu().to(torch.float64)
    else:
        want = torch.full((T * T,), 1.0 / model.r_max, dtype=torch.float64)
    got = v.detach().cpu().to(torch.float64).reshape(-1)
    if got.numel() == 1:
        got = got.expand(T * T)
    if got.numel() != T * T or not torch.equal(got, want):
        if model.per_edge_type_cutoff is None:
            raise ValueError(f"load_reference_state_dict: {rk} holds per-edge-type cutoffs; build the model with the "
                             "checkpoint's per_edge_type_cutoff (without it the model computes a different function)")
        raise ValueError(f"load_reference_state_dict: {rk} does not match the model's per_edge_type_cutoff table "
                         f"(checkpoint cutoffs {(1.0 / got).tolist()}, model {model.per_edge_type_cutoff.reshape(-1).tolist()})")


def to_reference_state_dict(model, prefix: str = "model.func.") -> Dict[str, torch.Tensor]:
    """This model's parameters under the reference's names (e3nn buffers are not produced)."""
    inv = {v: k for k, v in _key_map(model).items()}
    out = {}
    for k, v in model.state_dict().items():
        if k in inv:
            if k in ("scales", "shifts") and v.numel() == 0:
                continue
            out[prefix + inv[k]] = v.detach().clone()
    return out


def load_reference_state_dict(model, ref_sd: Dict[str, torch.Tensor], strict: bool = True) -> Tuple[list, list]:
    """Load a reference (nequip) state dict into ``model``.  Returns (missing, unexpected) like
    ``torch.nn.Module.load_state_dict``; with ``strict`` both must be empty (ignored e3nn buffers aside)."""
    kmap = _key_map(model)
    own = model.state_dict()
    new, unexpected, used = {}, [], set()
    for rk, v in ref_sd.items():
        if rk == RMAX_RECIP_KEY or rk.endswith("." + RMAX_RECIP_KEY):
            _check_rmax_recip(model, v, rk)
            if "rmax_recip" in own:
                new["rmax_recip"] = own["rmax_recip"].clone()  # equal to the checkpoint's table
                used.add("rmax_recip")
            continue
        hit = [s for s in kmap if rk == s or rk.endswith("." + s)]
        if not hit:
            if not _IGNORED.search(rk):
                unexpected.append(rk)
            continue
        ok = kmap[max(hit, key=len)]
        t = own[ok]
        if ok in ("scales", "shifts"):
            v = v.reshape(-1, 1).to(torch.float64)
            if v.numel() == 1 and t.numel() > 1:
                v = v.expand_as(t).clone()
            if t.numel() == 0:  # the model was built without scale / shift: adopt the checkpoint's table
                getattr(model, ok).resize_(v.shape)
                t = getattr(model, ok)
        if tuple(v.shape) != tuple(t.shape):
            raise ValueError(f"load_reference_state_dict: {rk} has shape {tuple(v.shape)}, expected {tuple(t.shape)} ({ok})")
        new[ok] = v.to(t.dtype)
        used.add(ok)
    missing = [k for k in own if k not in used and not (k in ("scales", "shifts") and own[k].numel() == 0)]
    if strict and (missing or unexpected):
        raise KeyError(f"load_reference_state_dict: missing {missing}, unexpected {unexpected}")
    merged = dict(model.state_dict())
    merged.update(new)
    model.load_state_dict(merged)
    return missing, unexpected
