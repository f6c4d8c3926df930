"""End-to-end parity of the CUDA path: `aurora_b200.Aurora*.forward` / `rollout` on an H100 against
(a) golden outputs of the unmodified reference (tests/golden/model_*.npz, float64 reference) and
(b) the CPU oracle run live on the same seeded inputs.

Stated tolerance: the path computes with bf16 GEMM operands and fp32 accumulation / residuals /
statistics (the reference's autocast recipe).  Per variable, rel-mean-abs error
mean|out-ref| / mean|ref| must stay within the reference's own PER-VARIABLE acceptance budget for its
stored outputs (reference tests/test_model.py:45-61, `tests/fixtures.py:REF_TOL`): 1e-4 for 2t / msl / t / z,
5e-3 for winds, humidity and the variables the reference never pins; the measured values are printed."""

import dataclasses
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import fixtures as fx
from tests.golden.cases import MODEL_CASES

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
NAN_TOL = 5e-3

CLASS_OF = {"Aurora": "Aurora", "AuroraAirPollution": "AuroraAirPollution", "AuroraSmallPretrained": "AuroraSmallPretrained"}


def _build(cfg_name, cls_name, seed):
    import aurora_b200 as ab

    cfg = fx.CONFIGS[cfg_name]
    model = getattr(ab, cls_name)(**fx.our_kwargs(cfg, cls_name))
    assert dataclasses.replace(model.config, autocast=False) == cfg   # only `autocast` differs (see fx.our_kwargs)
    extra = fx.air_extra_specs(cfg) if cls_name == "AuroraAirPollution" else ()
    model.load_state_dict(fx.make_state_dict(cfg, seed=seed, extra=extra), strict=True)
    # goldens and the live oracle are CPU evaluations of the reference algorithm; its scale encoding depends on the
    # device's sin() in the last bit (see AuroraEngine._pos_scale_embed), so evaluate the encodings where they did
    model.encoding_device = "cpu"
    return cfg, model.to("cuda").eval()


@pytest.mark.parametrize("name", sorted(MODEL_CASES))
def test_forward_matches_reference_golden(name):
    cfg_name, cls_name, h, w, levels, bsz, step, seed = MODEL_CASES[name]
    cfg, model = _build(cfg_name, cls_name, seed)
    batch = fx.case_inputs(MODEL_CASES[name])[2]
    wave = cls_name == "AuroraWave"
    eng = model._get_engine()
    eng.taps = {}
    pred = model.forward(batch)
    torch.cuda.synchronize()
    taps, eng.taps = eng.taps, None
    gold = np.load(GOLD / f"model_{name}.npz")
    # stage-level taps of the reference (forward hooks on its encoder / backbone, float64): the engine's encoder output
    # and decoder input for the LAST batch element
    for tap in ("encoder", "backbone"):
        ref_tap = torch.from_numpy(gold[f"tap.{tap}"])[-1]
        err = fx.rel_mean_abs(taps[tap][-1].cpu(), ref_tap)
        assert err < 5e-3, (name, tap, err)
    assert pred.metadata.rollout_step == int(gold["meta.rollout_step"])
    assert pred.metadata.time[0].timestamp() == float(gold["meta.time0"])
    worst = 0.0
    for grp, d in (("surf", pred.surf_vars), ("atmos", pred.atmos_vars)):
        keys = [k[len(grp) + 1:] for k in gold.files if k.startswith(grp + ".")]
        assert sorted(keys) == sorted(d.keys())
        if wave:
            assert list(d.keys()) == keys  # dict order produced by the reference's hooks
        for k in keys:
            ref = torch.from_numpy(gold[f"{grp}.{k}"])
            out = d[k].cpu()
            assert out.shape == ref.shape and out.is_floating_point()
            if not wave:
                assert torch.isfinite(out).all(), (grp, k)
            # wave model: NaN marks an absent wave component (density head < 0.5); a logit within bf16 noise of 0
            # may flip, so the NaN masks must agree on all but NAN_TOL of the points; directions are compared
            # on the circle
            err, nan_mismatch = fx.field_error(out, ref, angle=wave and k in fx.WAVE_ANGLES)
            worst = max(worst, err)
            assert err < fx.tol_for(k) and nan_mismatch < NAN_TOL, (name, grp, k, err, nan_mismatch)
    print(f"[parity] {name}: worst rel-mean-abs {worst:.3e}")
    for k, v in pred.static_vars.items():
        assert torch.equal(v.cpu(), batch.crop(cfg.patch_size).static_vars[k])


def test_forward_matches_oracle_live_on_new_shape():
    """A shape that has no stored golden: 0.25-degree-like aspect, odd merge (patch_res (4, 9, 18))."""
    from oracle import aurora_oracle as O

    cfg, model = _build("tiny_lora", "Aurora", 11)
    batch = fx.make_batch(cfg, 37, 72, levels=fx.LEVELS13, b=1, seed=11, rollout_step=1)
    pred = model.forward(batch)
    with torch.inference_mode():
        ref = O.forward(cfg, fx.make_state_dict(cfg, seed=11), batch, dtype=torch.float32)
    for grp, d, r in (("surf", pred.surf_vars, ref.surf_vars), ("atmos", pred.atmos_vars, ref.atmos_vars)):
        for k in d:
            assert fx.rel_mean_abs(d[k].cpu(), r[k]) < fx.tol_for(k), (grp, k)


def test_rollout_matches_reference_golden():
    import aurora_b200 as ab

    cfg, model = _build("tiny_lora", "Aurora", 7)
    batch = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, b=1, seed=7)
    gold = np.load(GOLD / "rollout_tiny_lora.npz")
    for i, pred in enumerate(ab.rollout(model, batch, steps=3)):
        assert pred.metadata.rollout_step == int(gold[f"step{i}.rollout_step"]) == i + 1
        for k, v in pred.surf_vars.items():
            assert fx.rel_mean_abs(v.cpu(), torch.from_numpy(gold[f"step{i}.surf.{k}"])) < fx.tol_for(k) * (i + 1), (i, k)
        for k, v in pred.atmos_vars.items():
            assert fx.rel_mean_abs(v.cpu(), torch.from_numpy(gold[f"step{i}.atmos.{k}"])) < fx.tol_for(k) * (i + 1), (i, k)


def test_wave_rollout_matches_oracle_live():
    """AuroraWave through `rollout` (hook applied once to the initial state, NaN fields fed back as density
    channels, LoRA from the second step) against the CPU oracle on the same inputs."""
    import aurora_b200 as ab
    from oracle import aurora_oracle as O

    cfg, model = _build("tiny_wave", "AuroraWave", 9)
    sd = fx.make_state_dict(cfg, seed=9)
    batch = fx.make_wave_batch(cfg, 33, 64, seed=9, rollout_step=0, with_dwi=True)
    with torch.inference_mode():
        refs = list(O.rollout(cfg, sd, batch, steps=2, dtype=torch.float32, variant="wave", variant_args=fx.WAVE_ARGS))
    for i, pred in enumerate(ab.rollout(model, batch, steps=2)):
        assert pred.metadata.rollout_step == i + 1
        assert list(pred.surf_vars) == list(refs[i].surf_vars)
        for grp, d, r in (("surf", pred.surf_vars, refs[i].surf_vars), ("atmos", pred.atmos_vars, refs[i].atmos_vars)):
            for k in d:
                err, nan_mismatch = fx.field_error(d[k].cpu(), r[k], angle=k in fx.WAVE_ANGLES)
                assert err < fx.tol_for(k) * (i + 1) and nan_mismatch < NAN_TOL * (i + 1), (i, grp, k, err, nan_mismatch)


def test_no_cpu_path():
    import aurora_b200 as ab

    cfg = fx.CONFIGS["tiny"]
    model = ab.Aurora(**fx.our_kwargs(cfg))
    with pytest.raises(RuntimeError, match="CUDA"):
        model.forward(fx.make_batch(cfg, 17, 32, levels=fx.LEVELS4))


def test_cuda_graph_replay_is_bit_identical_to_eager():
    """`model.use_cuda_graph`: capture once, replay on new inputs; same bits as the eager launches."""
    cfg, model = _build("tiny_lora", "Aurora", 13)
    b1 = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, b=1, seed=13)
    b2 = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, b=1, seed=14)
    e1 = {k: v.clone() for k, v in model.forward(b1).atmos_vars.items()}
    e2 = {k: v.clone() for k, v in model.forward(b2).atmos_vars.items()}
    model.use_cuda_graph = True
    g1 = {k: v.clone() for k, v in model.forward(b1).atmos_vars.items()}   # capture
    g2 = {k: v.clone() for k, v in model.forward(b2).atmos_vars.items()}   # replay with other inputs
    g1b = {k: v.clone() for k, v in model.forward(b1).atmos_vars.items()}  # replay again
    for k in e1:
        assert torch.equal(e1[k], g1[k]) and torch.equal(e2[k], g2[k]) and torch.equal(e1[k], g1b[k]), k


def test_sharded_step_replays_from_graph_segments():
    """A latitude-sharded step under `use_cuda_graph` is captured as graph segments with the halo exchanges issued
    eagerly between them.  On one GPU (world size 1) the band is the whole grid and the halo wraps onto itself, so
    the segmented replay must reproduce the eager sharded step and the plain forward bit for bit."""
    cfg, model = _build("tiny_lora", "Aurora", 17)
    # patch_res (4, 48, 64): full 144-token windows at all three stages (the wgmma slab kernel)
    b1 = fx.make_batch(cfg, 192, 256, levels=fx.LEVELS4, b=1, seed=17, rollout_step=1)
    b2 = fx.make_batch(cfg, 192, 256, levels=fx.LEVELS4, b=1, seed=18, rollout_step=1)
    plain = {k: v.clone() for k, v in model.forward(b1).atmos_vars.items()}
    eager1 = {k: v.clone() for k, v in model.forward(b1, sharded=True).atmos_vars.items()}
    eager2 = {k: v.clone() for k, v in model.forward(b2, sharded=True).atmos_vars.items()}
    model.use_cuda_graph = True
    g1 = {k: v.clone() for k, v in model.forward(b1, sharded=True).atmos_vars.items()}   # capture + first replay
    g2 = {k: v.clone() for k, v in model.forward(b2, sharded=True).atmos_vars.items()}   # replay, other inputs
    g1b = {k: v.clone() for k, v in model.forward(b1, sharded=True).atmos_vars.items()}
    entry = next(e for sig, e in model._engine._graphs.items() if sig[-2])  # the sharded signature
    n_graphs = sum(isinstance(i, torch.cuda.CUDAGraph) for i in entry["items"])
    assert n_graphs == 12 + 1 and len(entry["items"]) == 2 * 12 + 1  # 12 Swin blocks -> 12 exchanges, 13 segments
    for k in plain:
        assert torch.equal(plain[k], eager1[k]), k
        assert torch.equal(eager1[k], g1[k]) and torch.equal(eager2[k], g2[k]) and torch.equal(eager1[k], g1b[k]), k


def _pin(batch):
    from aurora_b200 import Batch

    pin = lambda d: {k: v.contiguous().pin_memory() for k, v in d.items()}  # noqa: E731
    return Batch(pin(batch.surf_vars), pin(batch.static_vars), pin(batch.atmos_vars), batch.metadata)


@pytest.mark.parametrize("cfg_name,cls_name,h,w,levels", [
    ("tiny_lora", "Aurora", 33, 64, fx.LEVELS4),            # 33 rows: cropped on the device, kernels read the copies
    ("tiny_lora", "Aurora", 32, 64, fx.LEVELS4),            # no crop: kernels read the upload buffers themselves
    ("tiny_air", "AuroraAirPollution", 48, 90, fx.LEVELS13),  # + previous-state pointers into the upload buffers
])
def test_pinned_host_batches_take_the_overlapped_upload_and_give_the_same_bits(cfg_name, cls_name, h, w, levels):
    """Batches in pinned host memory are uploaded on a copy stream into two alternating device buffer sets
    (`AuroraEngine._upload_pinned`); five back-to-back steps on different inputs — no synchronisation in between, so
    uploads overlap the previous step's kernels and both buffer sets are reused — must equal the pageable-memory
    path bit for bit, and predictions must not alias the upload buffers."""
    cfg, model = _build(cfg_name, cls_name, 23)
    batches = [fx.make_batch(cfg, h, w, levels=levels, b=1, seed=40 + i, rollout_step=i % 2) for i in range(5)]
    want = []
    for b in batches:
        p = model.forward(b)
        want.append(({k: v.clone() for k, v in p.surf_vars.items()}, {k: v.clone() for k, v in p.atmos_vars.items()},
                     {k: v.clone() for k, v in p.static_vars.items()}))
    pinned = [_pin(b) for b in batches]
    torch.cuda.synchronize()
    preds = [model.forward(b) for b in pinned]          # no sync between the steps
    torch.cuda.synchronize()
    assert model._engine._h2d is not None and all(s["busy"] is not None for s in model._engine._h2d["slots"])
    for p, (ws, wa, wst) in zip(preds, want):
        for k in ws:
            assert torch.equal(p.surf_vars[k], ws[k]), k
        for k in wa:
            assert torch.equal(p.atmos_vars[k], wa[k]), k
        for k in wst:
            assert torch.equal(p.static_vars[k], wst[k]), k


def test_cuda_graph_replay_follows_a_moved_grid():
    """Same shapes, other lat / lon (a moved regional domain): the position / scale embeddings are inputs of the
    captured graph like the Batch fields, so the replay must match the eager step on the new grid."""
    import dataclasses

    from aurora_b200 import Metadata

    cfg, model = _build("tiny_lora", "Aurora", 13)
    b1 = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, b=1, seed=13)
    md = b1.metadata
    moved = dataclasses.replace(b1, metadata=Metadata(lat=md.lat * 0.5 + 10.0, lon=(md.lon * 0.5 + 40.0) % 360.0,
                                                     time=md.time, atmos_levels=md.atmos_levels,
                                                     rollout_step=md.rollout_step))
    e1 = {k: v.clone() for k, v in model.forward(b1).atmos_vars.items()}
    e2 = {k: v.clone() for k, v in model.forward(moved).atmos_vars.items()}
    assert any(not torch.equal(e1[k], e2[k]) for k in e1)  # the grid matters
    model.use_cuda_graph = True
    g1 = model.forward(b1).atmos_vars        # capture
    g2 = model.forward(moved).atmos_vars     # replay on the moved grid
    g1b = model.forward(b1).atmos_vars       # and back
    for k in e1:
        assert torch.equal(e1[k], g1[k]) and torch.equal(e2[k], g2[k]) and torch.equal(e1[k], g1b[k]), k


@pytest.mark.parametrize("lora_mode", ["single", "all"])
def test_graph_rollout_yields_independent_predictions(lora_mode):
    """`list(rollout(...))` under `use_cuda_graph`: every entry keeps its own step's data (predictions are copies of the
    graph's static buffers), two consecutive roll-outs of 8 steps agree with the eager roll-out bit for bit — in
    `lora_mode="all"` that runs 8 different merged weight sets through graphs captured during the first roll-out."""
    import dataclasses

    import aurora_b200 as ab

    cfg = dataclasses.replace(fx.CONFIGS["tiny_lora"], lora_mode=lora_mode)
    model = ab.Aurora(**fx.our_kwargs(cfg))
    model.load_state_dict(fx.make_state_dict(cfg, seed=19), strict=True)
    model = model.to("cuda").eval()
    batch = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, b=1, seed=19)
    eager = [{k: v.clone() for k, v in p.atmos_vars.items()} for p in ab.rollout(model, batch, steps=8)]
    assert not torch.equal(eager[3]["t"], eager[7]["t"])
    model.use_cuda_graph = True
    for _ in range(2):
        preds = list(ab.rollout(model, batch, steps=8))
        assert [p.metadata.rollout_step for p in preds] == list(range(1, 9))
        for i, p in enumerate(preds):
            for k, v in p.atmos_vars.items():
                assert torch.equal(v, eager[i][k]), (i, k)


def test_whole_block_entry_point_equals_the_per_kernel_path():
    """`ab_swin_block` (one C call per Swin block: csrc/block.cu) issues exactly the launches the per-kernel path issues
    from Python — same bits, fewer calls; also with the skip-concatenation destination (fp16 halves of the decoder
    input) and for a zero-padded stage."""
    from aurora_b200 import cabi

    cfg, model = _build("tiny_lora", "Aurora", 29)
    batch = fx.make_batch(cfg, 192, 256, levels=fx.LEVELS4, b=1, seed=29, rollout_step=1)
    eng = model._get_engine()
    assert eng.block_entry
    model.forward(batch)   # packs weights and caches the location-independent vectors (one-time launches)
    n0 = cabi.launch_count()
    fused = model.forward(batch)
    n_fused = cabi.launch_count() - n0
    eng.block_entry = False
    n0 = cabi.launch_count()
    plain = model.forward(batch)
    n_plain = cabi.launch_count() - n0
    assert n_fused == n_plain  # same kernels, only the host-side call count differs
    for k in plain.atmos_vars:
        assert torch.equal(plain.atmos_vars[k], fused.atmos_vars[k]), k
    for k in plain.surf_vars:
        assert torch.equal(plain.surf_vars[k], fused.surf_vars[k]), k
    # ... and the whole backbone replayed from its recorded operation list (ONE ab_run_ops call per step) against
    # one ab_swin_block call per block: the forward above used the plan (eng.use_program), now without it
    assert eng.use_program and len(eng._programs) == 1
    eng.block_entry, eng.use_program = True, False
    n0 = cabi.launch_count()
    per_block = model.forward(batch)
    assert cabi.launch_count() - n0 == n_plain
    for k in plain.atmos_vars:
        assert torch.equal(per_block.atmos_vars[k], fused.atmos_vars[k]), k
    # the plan follows new inputs (it bakes buffer addresses, not values) and other roll-out steps get their own plan
    eng.use_program = True
    b2 = fx.make_batch(cfg, 192, 256, levels=fx.LEVELS4, b=1, seed=30, rollout_step=1)
    with_plan = {k: v.clone() for k, v in model.forward(b2).atmos_vars.items()}
    eng.use_program = False
    without = model.forward(b2).atmos_vars
    for k in with_plan:
        assert torch.equal(with_plan[k], without[k]), k


def test_stage_seams_backbone_forward_and_hooks():
    """`model.backbone.forward(x, lead_time, rollout_step, patch_res)` has the reference's signature (swin3d.py:884-890)
    and runs on the engine; forward hooks on `model.encoder` / `model.backbone` receive the stage outputs of
    `model.forward`, as the reference's parity tooling (tests/golden/make_golden.py) uses them.  The backbone called
    through the seam on the hooked encoder output reproduces the hooked backbone output, and both match the reference's
    stored taps."""
    from datetime import timedelta

    name = "tiny_lora_60x120_b2"
    cfg_name, cls_name, h, w, levels, bsz, step, seed = MODEL_CASES[name]
    cfg, model = _build(cfg_name, cls_name, seed)
    batch = fx.case_inputs(MODEL_CASES[name])[2]
    got = {}
    h1 = model.encoder.register_forward_hook(lambda m, i, o: got.__setitem__("encoder", o.clone()))
    h2 = model.backbone.register_forward_hook(lambda m, i, o: got.__setitem__("backbone", o.clone()))
    pred = model.forward(batch)
    h1.remove(), h2.remove()
    plain = model.forward(batch)   # no hooks: the fused path; same bits
    for k in plain.atmos_vars:
        assert torch.equal(plain.atmos_vars[k], pred.atmos_vars[k]), k
    gold = np.load(GOLD / f"model_{name}.npz")
    assert got["encoder"].shape == gold["tap.encoder"].shape and got["backbone"].shape == gold["tap.backbone"].shape
    for tap in ("encoder", "backbone"):
        assert fx.rel_mean_abs(got[tap].cpu(), torch.from_numpy(gold[f"tap.{tap}"])) < 5e-3, tap
    p = cfg.patch_size
    patch_res = (cfg.latent_levels, (h - h % p) // p, w // p)
    out = model.backbone(got["encoder"], timedelta(hours=6), step, patch_res)
    assert out.shape == got["backbone"].shape and out.dtype == torch.float32
    # the seam rounds its fp32 input to bf16 like the engine does after the encoder: identical arithmetic
    assert fx.rel_mean_abs(out.cpu(), got["backbone"].cpu()) < 1e-3
    with pytest.raises(NotImplementedError):
        model.backbone(got["encoder"], timedelta(hours=12), step, patch_res)
    with pytest.raises(NotImplementedError):
        model.encoder(batch, timedelta(hours=6))
