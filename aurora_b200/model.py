"""`Aurora` and its presets: same constructor arguments, ``state_dict`` keys, ``forward`` / checkpoint
methods as the reference (`aurora/model/aurora.py:40-643`), with the forward pass executed by the
sm_90a engine (``aurora_b200/engine.py``) instead of PyTorch modules.

The modules here are parameter containers only: they own fp32 ``nn.Parameter`` tensors under the
reference's names so that ``load_state_dict`` / ``load_checkpoint_local`` accept the reference's
checkpoints, and ``.to("cuda")`` moves them.  All computation happens in ``AuroraEngine``.
"""

from __future__ import annotations

import dataclasses
import warnings
import weakref
from datetime import timedelta
from typing import Optional

import torch
from torch import nn

from aurora_b200.batch import Batch
from aurora_b200.spec import ModelConfig, init_state_dict, param_specs

__all__ = [
    "Aurora", "AuroraPretrained", "AuroraSmallPretrained", "AuroraSmall", "Aurora12hPretrained", "AuroraHighRes",
    "AuroraAirPollution", "AuroraWave",
]


class _ParamNode(nn.Module):
    """A bare container; children are created on demand from dotted parameter names."""

    def put(self, path: list[str], value: torch.Tensor) -> None:
        node = self
        for part in path[:-1]:
            if part not in node._modules:
                node.add_module(part, _ParamNode())
            node = node._modules[part]
        node.register_parameter(path[-1], nn.Parameter(value, requires_grad=False))


class _BackboneSeam(_ParamNode):
    """`model.backbone`: the parameters of the reference's `Swin3DTransformerBackbone` under the same names, and its
    `forward` signature (swin3d.py:884-890) routed into the engine.  `Aurora.forward` itself runs the fused path and does
    not go through this method, but forward hooks registered here (and on `model.encoder`) are honoured: they are
    called with the stage's output, as for the reference's modules."""

    def forward(self, x: torch.Tensor, lead_time: timedelta, rollout_step: int, patch_res) -> torch.Tensor:
        owner = self.__dict__["_owner"]()
        if not owner.autocast:
            raise NotImplementedError("aurora_b200 has no fp32-exact mode: construct the model with autocast=True")
        return owner._get_engine().backbone_forward(x, lead_time, rollout_step, patch_res)


class _EncoderSeam(_ParamNode):
    """`model.encoder`: parameter container; forward hooks registered on it receive the encoder output (B, L, D) of
    every `Aurora.forward` call.  Its own `forward` is not offered: the encoder is fused with `Batch.normalise` and the
    variant hooks inside the patch loader (csrc/patch_io.cu), so there is no stand-alone "normalised Batch in" entry."""

    def forward(self, *a, **k):
        raise NotImplementedError(
            "aurora_b200 fuses normalisation and the encoder's patch embedding; run model.forward(batch) and read the "
            "encoder output with a forward hook on model.encoder")


_SEAMS = {"backbone": _BackboneSeam, "encoder": _EncoderSeam}


class Aurora(nn.Module):
    """The Aurora model (1.3 B parameter configuration by default), running on H100 (sm_90a) kernels.

    Constructor arguments: see `aurora/model/aurora.py:55-178`; they are stored in ``self.config``.
    """

    default_checkpoint_repo = "microsoft/aurora"
    default_checkpoint_name = "aurora-0.25-finetuned.ckpt"
    default_checkpoint_revision = "0be7e57c685dac86b78c4a19a3ab149d13c6a3dd"
    _variant = "base"

    def __init__(self, *, surf_stats: Optional[dict[str, tuple[float, float]]] = None, autocast: bool = False,
                 bf16_mode: bool = False, _init_seed: Optional[int] = None, _init: str = "reference", **kw) -> None:
        super().__init__()
        if surf_stats:
            warnings.warn(
                f"The normalisation statics for the following surface-level variables are manually "
                f"adjusted: {', '.join(sorted(surf_stats.keys()))}. Please ensure that this is right!",
                stacklevel=2,
            )
        if bf16_mode and not autocast:
            warnings.warn("`bf16_mode` was removed; it now activates `autocast`.", stacklevel=2)
            autocast = True
        for name in ("surf_vars", "static_vars", "atmos_vars", "window_size", "encoder_depths", "encoder_num_heads",
                     "decoder_depths", "decoder_num_heads", "level_condition", "separate_perceiver",
                     "modulation_heads", "positive_surf_vars", "positive_atmos_vars"):
            if name in kw and kw[name] is not None:
                kw[name] = tuple(kw[name])
        self.config = ModelConfig(
            surf_stats=tuple(sorted((k, tuple(v)) for k, v in surf_stats.items())) if surf_stats else None,
            autocast=autocast, bf16_mode=bf16_mode, **kw,
        )
        cfg = self.config
        assert sum(cfg.encoder_depths) == sum(cfg.decoder_depths)
        # attributes the reference exposes
        self.surf_vars, self.atmos_vars = cfg.surf_vars, cfg.atmos_vars
        self.patch_size = cfg.patch_size
        self.surf_stats = dict(surf_stats) if surf_stats else dict()
        self.max_history_size = cfg.max_history_size
        self.timestep = cfg.timestep
        self.use_lora = cfg.use_lora
        self.positive_surf_vars, self.positive_atmos_vars = cfg.positive_surf_vars, cfg.positive_atmos_vars
        self.clamp_at_first_step = cfg.clamp_at_first_step
        self.autocast = autocast

        if _init == "empty":  # benchmarks fill the parameters themselves (on the device)
            for key, shape, _kind in list(param_specs(cfg)) + list(self._extra_specs()):
                self._put(key, torch.empty(shape, dtype=torch.float32))
        else:
            for key, value in init_state_dict(cfg, seed=_init_seed, extra=self._extra_specs()).items():
                self._put(key, value)
        self._engine = None
        self._engine_sig = None
        self.encoding_device: Optional[str] = None
        """Device on which the position / scale encodings are evaluated; None = the parameters' device, which is what
        the reference does (`batch.to(device)` moves lat / lon, aurora.py:281).  The reference's scale encoding is
        device-dependent in its high-frequency features (float32 cancellation in the patch area, see
        `AuroraEngine._pos_scale_embed`); set "cpu" to reproduce a reference that ran on the CPU."""
        self.halo_mode = "auto"
        """str: transport of the halo exchange in `forward(batch, sharded=True)`: "peer" (kernels storing into the
        neighbouring GPUs' memory over NVLink, inside the step's CUDA graph), "nccl" (NCCL send / recv from the host),
        "auto" = "peer" whenever more than one rank takes part."""
        self.use_cuda_graph = False
        """bool: replay each forward step from a captured CUDA graph (one capture per input signature).  Predictions
        are copies of the graph's static output buffers, so they stay valid like the reference's."""

    # -- parameter tree ---------------------------------------------------------------------------
    def _extra_specs(self):
        return ()

    def _variant_args(self) -> dict:
        return {}

    def _apply(self, fn, *a, **k):  # .to() / .cuda() / .float(): parameters may be re-created
        self.__dict__.pop("_plist", None)
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self.__dict__.pop("_plist", None)
        return super().load_state_dict(*a, **k)

    def _put(self, key: str, value: torch.Tensor) -> None:
        self.__dict__.pop("_plist", None)
        path = key.split(".")
        if path[0] not in self._modules:
            node = _SEAMS.get(path[0], _ParamNode)()
            node.__dict__["_owner"] = weakref.ref(self)
            self.add_module(path[0], node)
        self._modules[path[0]].put(path[1:], value)

    # -- forward ----------------------------------------------------------------------------------
    def _get_engine(self):
        from aurora_b200.engine import AuroraEngine

        # (address, version) of every parameter: a new engine is packed whenever a weight moved or was written to.
        # The parameter list itself is cached (walking the module tree costs ~2 ms per forward on the 1.3 B model).
        plist = self.__dict__.get("_plist")
        if plist is None:
            plist = self.__dict__["_plist"] = [p for _, p in self.named_parameters()]
        sig = tuple((p.data_ptr(), p._version) for p in plist)
        if self._engine is None or sig != self._engine_sig:
            params = dict(self.named_parameters())
            p0 = next(iter(params.values()))
            if p0.dtype != torch.float32:
                raise NotImplementedError(
                    f"aurora_b200 keeps fp32 master parameters and computes with bf16 operands / fp32 accumulation; "
                    f"parameters of dtype {p0.dtype} are not supported")
            self._engine = AuroraEngine(self.config, {k: v.data for k, v in params.items()}, variant=self._variant,
                                        variant_args=self._variant_args())
            self._engine_sig = sig
        self._engine.use_cuda_graph = bool(self.use_cuda_graph)
        self._engine.halo_mode = self.halo_mode
        if self._engine.encoding_device != self.encoding_device:
            self._engine.encoding_device = self.encoding_device
            self._engine._grid_cache = None
        return self._engine

    def forward(self, batch: Batch, sharded: bool = False) -> Batch:
        """Forward pass: one model time step (`aurora.py:265-392`).

        `sharded=True` (one process per GPU under `torch.distributed`): every rank passes the same batch and
        gets back ITS latitude band of the prediction (see `aurora_b200/sharding.py`; `gather_bands` rebuilds
        full fields)."""
        if not self.autocast:
            # The reference's default (`autocast=False`, aurora.py:84) is a pure fp32 forward.  Hopper has no fp32
            # tensor-core path and this engine has no 3-pass split mode: it always computes with 16-bit operands and
            # fp32 accumulation, the reference's `autocast=True` recipe (aurora.py:327-343).  Running that under a
            # flag that promises fp32 would be a silent precision change, so it is refused.
            raise NotImplementedError(
                "aurora_b200 computes with bf16 / fp16 tensor-core operands and fp32 accumulation (the reference's "
                "`autocast=True` recipe) and has no fp32-exact mode: construct the model with `autocast=True` (or set "
                "`model.autocast = True`) to run it.")
        batch = self.batch_transform_hook(batch)
        eng = self._get_engine()
        hooked = [(nm, m) for nm, m in (("encoder", self._modules.get("encoder")), ("backbone", self._modules.get("backbone")))
                  if m is not None and m._forward_hooks]
        if not hooked:
            return eng.forward(batch, sharded=sharded)
        # forward hooks on the stage seams (the reference's parity tooling taps `model.encoder` / `model.backbone` this
        # way): run with stage taps and hand every hook the stage OUTPUT, (B, L, D) / (B, L, 2 D) float32
        saved, eng.taps = eng.taps, {}
        graph, eng.use_cuda_graph = eng.use_cuda_graph, False
        try:
            pred = eng.forward(batch, sharded=sharded)
            taps = eng.taps
        finally:
            eng.taps, eng.use_cuda_graph = saved, graph
        for nm, mod in hooked:
            out = torch.stack(taps[nm], 0)
            for hook in list(mod._forward_hooks.values()):
                hook(mod, (), out)
        return pred

    def batch_transform_hook(self, batch: Batch) -> Batch:
        return batch

    # -- checkpoints ------------------------------------------------------------------------------
    def load_checkpoint(self, repo: Optional[str] = None, name: Optional[str] = None,
                        revision: Optional[str] = None, strict: bool = True) -> None:
        """Download a checkpoint from HuggingFace and load it (`aurora.py:409-430`)."""
        try:
            from huggingface_hub import hf_hub_download
        except ImportError as e:  # pragma: no cover
            raise RuntimeError("huggingface_hub is required for load_checkpoint; use load_checkpoint_local") from e
        path = hf_hub_download(repo_id=repo or self.default_checkpoint_repo,
                               filename=name or self.default_checkpoint_name,
                               revision=revision or self.default_checkpoint_revision)
        self.load_checkpoint_local(path, strict=strict)

    def load_checkpoint_local(self, path: str, strict: bool = True) -> None:
        """Load a checkpoint file written for the reference (`aurora.py:432-456`)."""
        device = next(self.parameters()).device
        d = torch.load(path, map_location=device, weights_only=True)
        d = self._adapt_checkpoint(d)
        current = d["encoder.surf_token_embeds.weights.2t"].shape[2]
        if self.max_history_size > current:
            self.adapt_checkpoint_max_history_size(d)
        elif self.max_history_size < current:
            raise AssertionError(
                f"Cannot load checkpoint with `max_history_size` {current} "
                f"into model with `max_history_size` {self.max_history_size}.")
        self.load_state_dict(d, strict=strict)

    def _adapt_checkpoint(self, d: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
        """Bring a published checkpoint file to the current key layout (`aurora.py:458-467`,
        `aurora/model/compat.py:19-78`); a no-op for checkpoints already in that layout."""
        from aurora_b200 import compat

        return compat.adapt_pretrained(self.patch_size, d)

    def adapt_checkpoint_max_history_size(self, checkpoint: dict[str, torch.Tensor]) -> None:
        """Zero-extend the history dimension of the patch-embedding weights (`aurora.py:469-504`)."""
        for name, weight in list(checkpoint.items()):
            if name.startswith("encoder.surf_token_embeds.weights.") or name.startswith(
                    "encoder.atmos_token_embeds.weights."):
                if not (weight.shape[2] <= self.max_history_size):
                    raise AssertionError(
                        f"Cannot load checkpoint with `max_history_size` {weight.shape[2]} "
                        f"into model with `max_history_size` {self.max_history_size}.")
                new = torch.zeros((weight.shape[0], 1, self.max_history_size, weight.shape[3], weight.shape[4]),
                                  device=weight.device, dtype=weight.dtype)
                new[:, :, : weight.shape[2]] = weight
                checkpoint[name] = new

    def configure_activation_checkpointing(self, *a, **k) -> None:
        raise NotImplementedError(
            "Activation checkpointing (aurora.py:506-547) is a training feature; aurora_b200 is inference-only")


class AuroraPretrained(Aurora):
    default_checkpoint_name = "aurora-0.25-pretrained.ckpt"

    def __init__(self, *, use_lora: bool = False, **kw) -> None:
        super().__init__(use_lora=use_lora, **kw)


class AuroraSmallPretrained(Aurora):
    """Small configuration (aurora.py:568-598)."""

    default_checkpoint_name = "aurora-0.25-small-pretrained.ckpt"

    def __init__(self, *, encoder_depths=(2, 6, 2), encoder_num_heads=(4, 8, 16), decoder_depths=(2, 6, 2),
                 decoder_num_heads=(16, 8, 4), embed_dim: int = 256, num_heads: int = 8, use_lora: bool = False,
                 **kw) -> None:
        super().__init__(encoder_depths=encoder_depths, encoder_num_heads=encoder_num_heads,
                         decoder_depths=decoder_depths, decoder_num_heads=decoder_num_heads, embed_dim=embed_dim,
                         num_heads=num_heads, use_lora=use_lora, **kw)


AuroraSmall = AuroraSmallPretrained


class Aurora12hPretrained(Aurora):
    default_checkpoint_name = "aurora-0.25-12h-pretrained.ckpt"
    default_checkpoint_revision = "15e76e47b65bf4b28fd2246b7b5b951d6e2443b9"

    def __init__(self, *, timestep: timedelta = timedelta(hours=12), use_lora: bool = False, **kw) -> None:
        super().__init__(timestep=timestep, use_lora=use_lora, **kw)


class AuroraHighRes(Aurora):
    """0.1 degree configuration (aurora.py:624-643)."""

    default_checkpoint_name = "aurora-0.1-finetuned.ckpt"

    def __init__(self, *, patch_size: int = 10, encoder_depths=(6, 8, 8), decoder_depths=(8, 8, 6), **kw) -> None:
        super().__init__(patch_size=patch_size, encoder_depths=encoder_depths, decoder_depths=decoder_depths, **kw)


class AuroraAirPollution(Aurora):
    """CAMS air-pollution fine-tune (aurora.py:646-801): level-conditioned patch embeddings and heads,
    dynamic / atmospheric static variables, separate Perceiver, modulation heads, log-combiner inputs."""

    default_checkpoint_name = "aurora-0.4-air-pollution.ckpt"
    default_checkpoint_revision = "1764d5630a53d3d7a7d169ca335236fc343e4bfc"
    _variant = "air_pollution"

    _diff = ("pm1", "pm2p5", "pm10", "co", "tcco", "no", "tc_no", "no2", "tcno2", "so2", "tcso2", "go3", "gtco3")

    def __init__(
        self, *,
        surf_vars=("2t", "10u", "10v", "msl", "pm1", "pm2p5", "pm10", "tcco", "tc_no", "tcno2", "gtco3", "tcso2"),
        static_vars=("lsm", "z", "slt", "static_ammonia", "static_ammonia_log", "static_co", "static_co_log",
                     "static_nox", "static_nox_log", "static_so2", "static_so2_log"),
        atmos_vars=("z", "u", "v", "t", "q", "co", "no", "no2", "go3", "so2"),
        patch_size: int = 3, timestep: timedelta = timedelta(hours=12),
        level_condition=(50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925, 1000),
        dynamic_vars: bool = True, atmos_static_vars: bool = True,
        separate_perceiver=("co", "no", "no2", "go3", "so2"), modulation_heads=_diff,
        positive_surf_vars=("pm1", "pm2p5", "pm10", "tcco", "tc_no", "tcno2", "gtco3", "tcso2"),
        positive_atmos_vars=("co", "no", "no2", "go3", "so2"), simulate_indexing_bug: bool = True, **kw,
    ) -> None:
        super().__init__(
            surf_vars=surf_vars, static_vars=static_vars, atmos_vars=atmos_vars, patch_size=patch_size,
            timestep=timestep, level_condition=level_condition, dynamic_vars=dynamic_vars,
            atmos_static_vars=atmos_static_vars, separate_perceiver=separate_perceiver,
            modulation_heads=modulation_heads, positive_surf_vars=positive_surf_vars,
            positive_atmos_vars=positive_atmos_vars, simulate_indexing_bug=simulate_indexing_bug, **kw)

    def _extra_specs(self):
        cfg = self.config
        out = []
        for grp, names in (("surf_feature_combiner", cfg.positive_surf_vars),
                           ("atmos_feature_combiner", cfg.positive_atmos_vars)):
            for v in names:
                out.append((f"{grp}.{v}.weight", (1, 2), "half"))
                out.append((f"{grp}.{v}.bias", (1,), "zeros"))
        return out

    def _adapt_checkpoint(self, d: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
        from aurora_b200 import compat

        return compat.adapt_air_pollution(self.patch_size, Aurora._adapt_checkpoint(self, d))


_WAVE_VARS = (("swh", "mwd", "mwp", "pp1d", "shww", "mdww", "mpww", "shts", "mdts", "mpts")
              + ("swh1", "mwd1", "mwp1", "swh2", "mwd2", "mwp2", "wind", "10u_wave", "10v_wave"))


class AuroraWave(Aurora):
    """HRES-WAM ocean-wave fine-tune (aurora.py:804-920).  Wave variables that are absent are NaN in the data:
    every such variable gets a `<name>_density` presence channel, directions are modelled as sine / cosine.
    The channel construction runs inside the patch loader, the inverse (atan2, density -> NaN on the wave
    model mask `wmb`) inside the un-patchify kernel (`csrc/patch_io.cu`)."""

    default_checkpoint_name = "aurora-0.25-wave.ckpt"
    default_checkpoint_revision = "74598e8c65d53a96077c08bb91acdfa5525340c9"
    _variant = "wave"

    def __init__(
        self, *,
        surf_vars=("2t", "10u", "10v", "msl") + _WAVE_VARS,
        static_vars=("lsm", "z", "slt", "wmb", "lat_mask"),
        lora_mode: str = "from_second", stabilise_level_agg: bool = True,
        density_channel_surf_vars=_WAVE_VARS,
        angle_surf_vars=("mwd", "mdww", "mdts", "mwd1", "mwd2"), **kw,
    ) -> None:
        # the network models the sine, cosine and density versions of the variables (aurora.py:826-834)
        supplemented: tuple[str, ...] = ()
        for name in surf_vars:
            supplemented += (f"{name}_sin", f"{name}_cos") if name in angle_surf_vars else (name,)
            if name in density_channel_surf_vars:
                supplemented += (f"{name}_density",)
        super().__init__(surf_vars=supplemented, static_vars=static_vars, lora_mode=lora_mode,
                         stabilise_level_agg=stabilise_level_agg, **kw)
        self.density_channel_surf_vars = tuple(density_channel_surf_vars)
        self.angle_surf_vars = tuple(angle_surf_vars)

    def _variant_args(self) -> dict:
        return {"density_vars": self.density_channel_surf_vars, "angle_vars": self.angle_surf_vars}

    def _adapt_checkpoint(self, d: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
        from aurora_b200 import compat

        return compat.adapt_wave(self.patch_size, Aurora._adapt_checkpoint(self, d))

    def batch_transform_hook(self, batch: Batch) -> Batch:
        """Host-side preparation of raw HRES-WAM fields, before normalisation (aurora.py:851-890): wind speed +
        direction -> components, and at the first step waves of (practically) zero height are marked absent."""
        surf = dict(batch.surf_vars)
        if "dwi" in surf and "wind" in surf:
            ang = torch.deg2rad(surf.pop("dwi"))
            surf["10u_wave"] = -surf["wind"] * torch.sin(ang)
            surf["10v_wave"] = -surf["wind"] * torch.cos(ang)
        if batch.metadata.rollout_step == 0:
            families = (("swh", ("mwd", "mwp", "pp1d")), ("shww", ("mdww", "mpww")), ("shts", ("mdts", "mdts")),
                        ("swh1", ("mwd1", "mwp1")), ("swh2", ("mwd2", "mwp2")))
            for height, others in families:
                absent = surf[height] < 1e-4
                if bool(absent.any()):
                    for name in (height,) + others:
                        surf[name] = surf[name].masked_fill(absent, float("nan"))
                        if name not in self.angle_surf_vars:
                            assert int((surf[name] < 1e-4).sum()) == 0
        return dataclasses.replace(batch, surf_vars=surf)
