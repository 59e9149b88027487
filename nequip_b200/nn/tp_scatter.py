"""Drop-in ``TensorProductScatter`` backed by the fused sm_90a kernels.

Mirrors, for the fused CUDA path, what the reference ships for its two third-party
kernel back-ends:

* ``OpenEquivarianceTensorProductScatter``  nequip/nn/_tp_scatter_oeq.py:4-57
* ``CuEquivarianceTensorProductScatter``    nequip/nn/_tp_scatter_cueq.py:66-122
* the ``enable_*`` model modifiers          nequip/nn/_tp_scatter_base.py:40-109

Constructor and ``forward`` signatures are exactly the base class's
(nequip/nn/_tp_scatter_base.py:10-38): ``(feature_irreps_in, irreps_edge_attr,
irreps_mid, instructions)`` and ``forward(x, edge_attr, edge_weight, edge_dst,
edge_src) -> [x.size(0), irreps_mid.dim]``.

When ``nequip`` (and hence e3nn) is importable the class subclasses the real
``TensorProductScatter`` -- keeping ``self.tp`` alive for state-dict compatibility,
as the reference's subclasses do -- and the modifier is attached to it so that
``nequip.model.modify`` / ``nequip-compile --modifiers enable_B200TensorProductScatter``
find it.  Without nequip the same class stands alone on ``torch.nn.Module``.
"""
from __future__ import annotations

import torch

from .. import ops
from .. import torch_ops  # registers torch.ops.nequip_b200.* (no native code is loaded by the import)
from ..codegen import GenOptions
from ..irreps import Irreps

try:  # the reference stack is optional at run time (absent in this container)
    from nequip.nn._tp_scatter_base import TensorProductScatter as _RefTensorProductScatter  # type: ignore

    _HAVE_NEQUIP = True
except Exception:  # pragma: no cover - exercised only where nequip is installed
    _RefTensorProductScatter = None
    _HAVE_NEQUIP = False


class TensorProductScatterInterface(torch.nn.Module):
    """The attribute contract of the reference base class (nequip/nn/_tp_scatter_base.py:10-33)
    minus the e3nn ``self.tp`` module, for use when nequip/e3nn are not installed."""

    def __init__(self, feature_irreps_in, irreps_edge_attr, irreps_mid, instructions) -> None:
        super().__init__()
        self.feature_irreps_in = feature_irreps_in
        self.irreps_edge_attr = irreps_edge_attr
        self.irreps_mid = irreps_mid
        self.instructions = instructions
        self.model_dtype = torch.get_default_dtype()


_Base = _RefTensorProductScatter if _HAVE_NEQUIP else TensorProductScatterInterface


class B200TensorProductScatter(_Base):
    _nequip_custom_ops_libs = ("nequip_b200",)

    def __init__(
        self,
        feature_irreps_in,
        irreps_edge_attr,
        irreps_mid,
        instructions,
        layout: str = "mul_ir",
    ) -> None:
        super().__init__(
            feature_irreps_in=feature_irreps_in,
            irreps_edge_attr=irreps_edge_attr,
            irreps_mid=irreps_mid,
            instructions=instructions,
        )
        # ^ with nequip installed the base class keeps `self.tp` (and its persistent buffers)
        # around so that state dicts load with or without this modifier applied
        # layout="mul_ir" is the reference's (e3nn) node-feature layout and the drop-in default;
        # "ir_mul" (channel-contiguous, what cuEquivariance uses, nequip/nn/_tp_scatter_cueq.py:107-122)
        # is used between our own kernels
        self.layout = layout
        # the signature is pure host logic; the kernel library is bound on first use, so that constructing a
        # model (e.g. to obtain a state dict for the CPU reference arm of bench.py) loads no native code
        from ..codegen import TPSignature

        self._sig = TPSignature(Irreps(feature_irreps_in), Irreps(irreps_edge_attr), Irreps(irreps_mid), list(instructions))
        self.weight_numel = self._sig.weight_numel
        self._plan_obj = None
        self._key = None

    @property
    def _plan(self):
        if self._plan_obj is None:
            s = self._sig
            self._plan_obj = ops.get_plan(s.irreps_in1, s.irreps_in2, s.irreps_out, s.instructions, GenOptions(layout=self.layout))
        return self._plan_obj

    @property
    def _plan_key(self) -> str:
        if self._key is None:
            self._key = torch_ops.register_plan(self._plan)
        return self._key

    def forward(self, x, edge_attr, edge_weight, edge_dst, edge_src):
        # one opaque ``torch.ops.nequip_b200.tp_scatter`` node (fake kernel + autograd of any order registered in
        # nequip_b200/torch_ops.py): traceable by make_fx / torch.compile / torch.export, usable in training.
        # explicit cast to account for AMP (as the OpenEquivariance subclass does)
        dt = self.model_dtype
        return torch.ops.nequip_b200.tp_scatter(x.to(dt), edge_attr.to(dt), edge_weight.to(dt), edge_dst, edge_src,
                                                self._plan_key)


def _factory(old):
    prev = torch.get_default_dtype()
    torch.set_default_dtype(old.model_dtype)
    try:
        new = B200TensorProductScatter(
            feature_irreps_in=old.feature_irreps_in,
            irreps_edge_attr=old.irreps_edge_attr,
            irreps_mid=old.irreps_mid,
            instructions=old.instructions,
        )
        if hasattr(old, "tp"):
            # reuse old.tp to preserve e3nn's compiled buffers (state-dict compatibility,
            # c.f. nequip/nn/_tp_scatter_base.py:71-74)
            new.tp = old.tp
    finally:
        torch.set_default_dtype(prev)
    return new


def _replace_submodules(model: torch.nn.Module, target_cls, factory) -> torch.nn.Module:
    """``nequip.nn.model_modifier_utils.replace_submodules`` (nequip/nn/model_modifier_utils.py:92-107)."""
    if isinstance(model, target_cls) and not isinstance(model, B200TensorProductScatter):
        return factory(model)
    for name, child in list(model.named_children()):
        new = _replace_submodules(child, target_cls, factory)
        if new is not child:
            setattr(model, name, new)
    return model


def enable_B200TensorProductScatter(model: torch.nn.Module) -> torch.nn.Module:
    """Model modifier: swap every ``TensorProductScatter`` for the fused sm_90a kernel.

    Same role as ``TensorProductScatter.enable_OpenEquivariance``
    (nequip/nn/_tp_scatter_base.py:40-77).  CPU models are rejected like the
    reference's ``unsupported_devices=["cpu"]``."""
    try:
        p = next(model.parameters())
        if p.device.type == "cpu" and not torch.cuda.is_available():
            raise RuntimeError("enable_B200TensorProductScatter: CUDA (sm_90a) device required")
    except StopIteration:
        pass
    return _replace_submodules(model, _Base if not _HAVE_NEQUIP else _RefTensorProductScatter, _factory)


if _HAVE_NEQUIP:  # pragma: no cover - exercised only where nequip is installed
    from nequip.nn.model_modifier_utils import model_modifier, replace_submodules  # type: ignore

    def _enable(cls, model):
        return replace_submodules(model, cls, _factory)

    _RefTensorProductScatter.enable_B200TensorProductScatter = model_modifier(
        persistent=False,
        private=False,
        unsupported_devices=["cpu"],
        supported_compile_modes=["compile", "aotinductor"],  # opaque torch.library op with a fake kernel
    )(classmethod(_enable))
