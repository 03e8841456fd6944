"""qfx_gemm_bf16 where its persistent schedule gives each CTA several tiles (tools/gemm_sched_check.py).

GPU (`-m gpu`): every case of the tool: each launch bit-identical to its one-tile-per-CTA reference and to itself run again, and
per tile and per row against fp64 (gemm_tile_check.run), at synthetic tile counts and at the launches a training step makes.

CPU, with tests/emu_lib.py's `gemm` standing in for the kernel:
  * the one-tile-per-CTA reference reproduces the full launch bit for bit for every epilogue: gates expanded per row where a slice
    starts inside a batch, ATTN_DO slices inside one sample at advanced joint offsets, ragged band sub-lists, the aliased ADD;
  * a GEMM that adds one ulp to one tile a CTA computes second, or computes one tile with the k-block count of the problem the CTA's
    previous tile belonged to, is flagged at exactly that tile (problem, m-tile, n-tile, CTA, position), and nothing else is;
  * the recorder, on a tiny-width emulated step of each model family, captures the call sites the GPU cases replay;
  * the synthetic plans give some CTA two tiles in every launch but the exactly-SMs control, reach every (epilogue, block_n) pair,
    the smem ring edges and streamed stores, and switch LoRA k-block counts between a CTA's tiles, at 132 and 114 SMs."""
import json
import os
import sys
import types

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, HERE)

import emu_lib as emu  # noqa: E402
import gemm_sched_check as gs  # noqa: E402
from glue_check import Checks  # noqa: E402


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(gs.CASES))
def test_gemm_schedule_case(name):
    r = gs.CASES[name]()
    print(f"GEMM-SCHED {name} " + json.dumps(r))
    assert not r["fail"], r["fail"]


# ------------------------------------------------------------------------------------------------------------------ CPU
def _band_honest(gemm):
    """emu_lib's gemm computes every row of a ragged problem; the kernel writes only the rows of its bands (and zero-fills the dead
    ones).  This wrapper restores every other row, so that band sub-lists are held to covering the rows they must."""
    def run(problems, N, K, **kw):
        keep = []
        for p in problems:
            if p.row_bands is None:
                continue
            M = p.A.shape[0]
            mine = torch.zeros(M, dtype=torch.bool)
            for s in p.row_bands.host_tiles:
                mine[s:s + 256] = True
            for lo, hi in p.row_bands.host_dead:
                mine[lo:hi] = True
            for o in (p.out, p.out2):
                if o is not None:
                    keep.append((o, ~mine, o[~mine].clone()))
        gemm(problems, N, K, **kw)
        for o, rows, v in keep:
            o[rows] = v
    return run


def _exact(probs):
    """operands on a 1/8 grid in [-4, 4]: every fp32 partial sum of the emulated GEMM is exact, so its bits do not depend on how the
    host BLAS blocks a launch of another M (the kernel's own k order is what the GPU cases hold fixed)"""
    for p in probs:
        for k in ("A", "B", "A2", "B2"):
            if p.get(k) is not None:
                p[k].copy_((p[k].float() * 8).round().clamp(-32, 32) / 8)
    return probs


def _lib(gemm):
    return types.SimpleNamespace(gemm_problem=emu.gemm_problem, gemm=gemm)


def _ragged(epi, tb, seed):
    """a pad-to-max row group of 4 samples x 700 rows (valid 700 / 100 / 0 / 420) next to a dense group: 7 bands, two dead ranges"""
    from qflux_b200 import lib
    R, valid = 700, [700, 100, 0, 420]
    tiles, dead = lib.RowBands.plan(valid, R)
    s = gs._spec(epi, tb, 128, [len(tiles) * 2, 3], 1, 128, kb2=(1, 0), seed=seed, rpb=R)
    s["probs"][0].update(M=R * len(valid), bands=(tuple(tiles), tuple(tuple(d) for d in dead)))
    return s


def _cpu_specs():
    out = []
    for epi, tb in gs.EPI_SETS:
        tn = 1 if epi == gs.EPI_ATTN_DO else 2
        out.append((f"{gs._epi_tag(epi, tb)}_dense", gs._spec(epi, tb, 128, [5, 3, 4], tn, 128, kb2=(1, 0, 2), seed=3)))
        if epi in (gs.EPI_BIAS, gs.EPI_GELU, gs.EPI_RESID_GATE, gs.EPI_DGELU, gs.EPI_ADD):
            out.append((f"{gs._epi_tag(epi, tb)}_ragged", _ragged(epi, tb, 5)))
    out.append(("add_alias", gs._spec(gs.EPI_ADD, True, 128, [5, 3], 2, 128, alias=True, seed=7)))
    return out


@pytest.mark.parametrize("tag,spec", _cpu_specs(), ids=[t for t, _ in _cpu_specs()])
def test_one_tile_per_cta_reference_reproduces_the_launch(tag, spec):
    """With 3 SMs every reference launch has at most 3 tiles: RESID_GATE slices start inside a 97-row batch (the gate goes in
    expanded per row), ATTN_DO slices cut inside samples at advanced joint offsets, ragged problems go in as band sub-lists."""
    calls = []
    gemm = _band_honest(emu.gemm)

    def counting(problems, N, K, **kw):
        calls.append([(p.A.shape[0], p.rows_per_batch, p.s_offset, None if p.row_bands is None else len(p.row_bands.host_tiles))
                      for p in problems])
        gemm(problems, N, K, **kw)
    probs = _exact(gs.build_probs(spec, "cpu"))
    c = Checks()
    sched = gs.invariance(c, tag, probs, spec["N"], spec["K"], gs._cfg(spec), 3, L=_lib(counting))
    assert not c.fail, c.fail
    assert sched.per_cta()[1] >= 3
    ref = calls[2:]
    assert len(ref) > len(probs) and all(len(x) == 1 for x in ref)
    assert all(gs.m_tiles(M, [0] * nb if nb else None) * sched.tn <= 3 for ((M, _, _, nb),) in ref)
    if spec["epi"] == gs.EPI_RESID_GATE and "dense" in tag:
        assert any(rpb == 1 for ((_, rpb, _, _),) in ref) and any(rpb == 97 for ((_, rpb, _, _),) in ref)
    if spec["epi"] == gs.EPI_ATTN_DO:
        offs = {(g["s_offset"], g["rows_per_batch"]) for g in spec["probs"]}
        assert any((so, rpb) not in offs for ((_, rpb, so, _),) in ref)  # slices inside a sample, at advanced offsets
    if "ragged" in tag:
        assert any(nb is not None and nb < len(spec["probs"][0]["bands"][0]) for ((_, _, _, nb),) in ref)


def _mutation_spec():
    """six problems whose LoRA k-block counts alternate (0, 2, 1, 3, 0, 2), three LoRA groups: 39 tiles on 8 CTAs"""
    return gs._spec(gs.EPI_BIAS, False, 128, [2, 3, 1, 4, 1, 2], 3, 128, kb2=(0, 2, 1, 3, 0, 2), lora_group_n=128, seed=11)


SMS = 8


def _tile_rows(p, mt):
    M = p.A.shape[0]
    if p.row_bands is None:
        return mt * 128, min(M, (mt + 1) * 128)
    s = p.row_bands.host_tiles[mt // 2] + (mt % 2) * 128
    return s, min(M, s + 128)


def _sched_of(problems, N, kw):
    return gs.Schedule([gs.m_tiles(p.A.shape[0], None if p.row_bands is None else p.row_bands.host_tiles) for p in problems], N,
                       kw["block_n"], SMS)


def test_mutation_one_ulp_in_a_later_tile_is_named():
    """One ulp added to one element of the tile CTA 3 computes second: the check names that tile and nothing else."""
    target = (3, 1)

    def gemm(problems, N, K, **kw):
        emu.gemm(problems, N, K, **kw)
        sc = _sched_of(problems, N, kw)
        t = target[0] + target[1] * sc.grid
        if t < sc.total:
            i, mt, nt = sc.decode(t)
            r0, _ = _tile_rows(problems[i], mt)
            o = problems[i].out
            o.view(torch.int16)[r0, nt * kw["block_n"]] += 1
    spec = _mutation_spec()
    probs = _exact(gs.build_probs(spec, "cpu"))
    c = Checks()
    sched = gs.invariance(c, "ulp", probs, spec["N"], spec["K"], gs._cfg(spec), SMS, L=_lib(gemm))
    i, mt, nt = sched.decode(target[0] + target[1] * sched.grid)
    assert c.res["ulp_bad_tiles"] == [[i, mt, nt, target[0], target[1]]], c.fail
    assert c.res["ulp_repeat_bad_tiles"] == []
    assert len(c.fail) == 1 and f"problem {i} m-tile {mt} n-tile {nt}" in c.fail[0] and f"CTA {target[0]} computes it as tile 1" in c.fail[0]


def test_mutation_previous_problems_k_block_count_is_named():
    """The first tile whose CTA's previous tile belongs to a problem with fewer LoRA k-blocks is computed with that count (a stage
    handed back one k-block early when kb_total changes): the check names that tile and nothing else."""
    def victim(problems, sc):
        for t in range(sc.grid, sc.total):
            i, _, _ = sc.decode(t)
            j, _, _ = sc.decode(t - sc.grid)
            if problems[j].kb2 < problems[i].kb2:
                return t, problems[j].kb2
        return None, None

    def gemm(problems, N, K, **kw):
        emu.gemm(problems, N, K, **kw)
        sc = _sched_of(problems, N, kw)
        t, kb2 = victim(problems, sc)
        if t is None:
            return
        i, mt, nt = sc.decode(t)
        p = problems[i]
        tmp = types.SimpleNamespace(**dict(vars(p), out=p.out.clone(), kb2=kb2))
        emu.gemm([tmp], N, K, **kw)
        r0, r1 = _tile_rows(p, mt)
        bn = kw["block_n"]
        p.out[r0:r1, nt * bn:(nt + 1) * bn] = tmp.out[r0:r1, nt * bn:(nt + 1) * bn]
    spec = _mutation_spec()
    probs = _exact(gs.build_probs(spec, "cpu"))
    c = Checks()
    sched = gs.invariance(c, "kb2", probs, spec["N"], spec["K"], gs._cfg(spec), SMS, L=_lib(gemm))
    t, _ = victim([types.SimpleNamespace(kb2=p.get("kb2", 0)) for p in probs], sched)
    assert t is not None and t >= sched.grid
    i, mt, nt = sched.decode(t)
    cta, pos, _ = sched.where(t)
    assert c.res["kb2_bad_tiles"] == [[i, mt, nt, cta, pos]], c.fail
    assert c.res["kb2_repeat_bad_tiles"] == [] and len(c.fail) == 1


TINY = {"qwen_edit": dict(tiny=dict(heads=2), cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2)),
        "flux_kontext": dict(tiny=dict(heads=2), cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2))}


@pytest.fixture()
def emu_installed():
    from qflux_b200 import lib
    restore = emu.install(lib)
    yield lib
    restore()


@pytest.mark.parametrize("config", list(TINY))
def test_recorder_captures_the_step_call_sites(emu_installed, config):
    """The launches the GPU cases replay, recorded from one emulated step of a one-block tiny-width model of each family."""
    B = 2
    launches, D, C_out, rp = gs.record(config, B, torch.device("cpu"), **TINY[config])
    kinds = {}
    for r in launches:
        kinds.setdefault(gs.site_kind(r, D, C_out, rp), []).append(r)
    need = {"qkv", "out_resid_gate", "mlp_up_gelu", "dgelu", "attn_do", "lora_u", "proj_out_fwd", "proj_out_dgrad"}
    need |= {"down_resid_gate"} if config.startswith("qwen") else {"s_out", "add_alias"}
    assert need <= set(kinds), sorted(kinds)
    assert any(r["lora_group_n"] == D and any(p["kb2"] > 0 for p in r["probs"]) for r in kinds["qkv"])
    for k in ("out_resid_gate", "down_resid_gate", "s_out"):
        for r in kinds.get(k, []):
            assert all(p["gate"] and p["resid"] for p in r["probs"])
            if config == "flux_kontext":  # the YAML targets put LoRA on the AdaLN linears: the un-gated output is kept
                assert all(p["out2"] for p in r["probs"])
    if config == "flux_kontext":
        assert "down_resid_gate" in kinds
    T, Limg = TINY[config]["cfg_update"]["T"], 2 * 16
    for r in kinds["attn_do"]:  # image rows at joint offset T, text rows at 0
        assert r["N"] == D and [(p["s_offset"], p["rows_per_batch"]) for p in r["probs"]] == [(T, Limg), (0, T)]
        assert all(p["attn"] == (B, D // 128, T + Limg) for p in r["probs"])
    assert all(r["N"] == rp and r["bn"] == 64 for r in kinds["lora_u"])
    if config == "flux_kontext":
        assert all(r["N"] == D and r["K"] == 5 * D for r in kinds["s_out"])
        assert all(r["N"] == D and r["K"] == 4 * D for r in kinds["add_alias"])
    for r in launches:  # every recorded launch replays on fresh operands
        spec = gs.replay_spec(r, 1)
        assert spec["N"] == r["N"] and [p["M"] for p in spec["probs"]] == [p["M"] for p in r["probs"]]


@pytest.mark.parametrize("sms", [132, 114])
def test_synthetic_plan_reaches_the_schedule_edges(sms):
    """Pure arithmetic: some CTA gets two tiles in every synthetic launch but the exactly-SMs control; every (epilogue, block_n)
    pair, each K edge of the smem ring and streamed stores per epilogue are reached; in the six-problem launches some CTA's next
    tile has another LoRA k-block count; every launch's n-tiles fit on the SMs, so its reference runs one tile per CTA."""
    plan = gs.plan(sms)
    pairs, stream, ks, switches = set(), set(), set(), 0
    for case, launches in plan.items():
        for tag, s, control in launches:
            sc = gs.Schedule([gs.m_tiles(p["M"]) for p in s["probs"]], s["N"], s["bn"], sms)
            lo, hi = sc.per_cta()
            assert control == (sc.total == sms), (case, tag)
            assert control or hi >= 2, (case, tag, sc.stats())
            assert sc.tn <= sms
            pairs.add((s["epi"], s["trans_b"], s["bn"]))
            if gs.stream_out([p["M"] for p in s["probs"]], s["N"], s["epi"]):
                stream.add((s["epi"], s["trans_b"]))
            if case.startswith("ring"):
                ks.add((s["bn"], s["K"]))
            if case == "switch":
                kb = [p["kb2"] for p in s["probs"]]
                assert len(set(kb)) == 4 and all(p["a2_col0"] > 0 for p in s["probs"] if p["kb2"])
                assert s["trans_b"] or s["lora_group_n"] > 0
                changes = sum(kb[sc.decode(t)[0]] != kb[sc.decode(t - sc.grid)[0]] for t in range(sc.grid, sc.total))
                assert changes > 0
                switches += 1
    assert pairs == {(e, t, b) for e, t in gs.EPI_SETS for b in gs.bns(e)}
    assert stream == set(gs.EPI_SETS)
    assert ks == {(b, k) for b, S in gs.STAGES.items() for k in (64, S * 64, S * 64 + 64, 4096)}
    assert switches == len(gs.EPI_SETS)
    assert sum(c for launches in plan.values() for _, _, c in launches) == sum(len(gs.bns(e)) for e, _ in gs.EPI_SETS)


def test_schedule_restates_the_kernel_decode():
    """The Qwen-Image-Edit B = 1 block GEMMs (352 text + 2048 image rows): 684 / 912 / 228 tiles for q|k|v, MLP up and out / down, and
    the MLP up's outputs stream past L2; tile t runs on CTA t % grid as its (t // grid)-th tile, problems in order inside each n-block."""
    for N, epi, tiles in ((9216, gs.EPI_BIAS, 684), (12288, gs.EPI_GELU, 912), (3072, gs.EPI_RESID_GATE, 228)):
        sc = gs.Schedule([gs.m_tiles(352), gs.m_tiles(2048)], N, gs.auto_bn(N, epi), 132)
        assert sc.total == tiles and sc.grid == 132
    assert gs.stream_out([352, 2048], 12288, gs.EPI_GELU) and not gs.stream_out([352, 2048], 3072, gs.EPI_RESID_GATE)
    sc = gs.Schedule([3, 16], 3072, 256, 132)
    assert [sc.decode(t) for t in (0, 2, 3, 18, 19, 227)] == [(0, 0, 0), (0, 2, 0), (1, 0, 0), (1, 15, 0), (0, 0, 1), (1, 15, 11)]
    assert sc.where(140) == (8, 1, 2) and sc.where(131) == (131, 0, 1) and sc.per_cta() == (1, 2)
    assert all(sc.tile(*sc.decode(t)) == t for t in range(sc.total))
