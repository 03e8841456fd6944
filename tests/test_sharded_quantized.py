"""Sharded NF4 / FP8 frozen weights (`shard_frozen_weights()` on a model built with frozen_weights="nf4" or "fp8", DESIGN.md §5):
every rank keeps 1/world of each block's packed code bytes, and a block is filled by gathering the shards into a staging slot and
expanding them into the ring's bf16 slot (sharding.ShardedCodes).

CPU (gloo worlds of 2 and 3, emulated kernels: tests/emu_lib.py + tests/nf4_ref.py + tests/fp8_ref.py): the gather only moves bytes
and the expansion is exact, so loss, prediction and the whole LoRA gradient equal the unsharded model of the same format bit for
bit on each rank's batch; the resident code bytes per rank are 1/world of the unsharded store (plus alignment padding) and the full
stacks are freed; the refusals.  GPU (`-m gpu`, one subprocess per case, tools/sharded_quant_check.py): two processes sharing one
H100 with the peer gather, bit for bit against an unsharded model of the same format, eager and CUDA-graph replayed."""
import os
import socket
import subprocess
import sys
import weakref

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
QWEN_TARGETS = ("to_q", "to_k", "to_v", "to_out.0", "add_q_proj", "img_mod.1", "txt_mod.1", "img_mlp.net.2", "txt_mlp.net.0.proj",
                "img_in", "txt_in")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _setup(rank, world, port):
    for p in (HERE, ROOT, os.path.join(ROOT, "qwen-image-finetune_b200")):
        sys.path.insert(0, p)
    import fp8_ref
    import nf4_ref
    from qflux_b200 import lib
    nf4_ref.install(lib)
    lib.fp8_expand = fp8_ref.fp8_expand
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _quantized(family, fmt):
    """A reduced quantized model of `fmt` ("nf4" / "fp8") and family: the same weights and adapter on every call and every rank."""
    import nf4_ref
    import test_activation_recompute as tar
    import test_fp8_weights as tfp
    src = tar._qwen(L=3, targets=QWEN_TARGETS) if family == "qwen" else tar._flux(nd=2, ns=3)
    base = {k.replace(".base_layer.", "."): v for k, v in src.state_dict().items() if ".lora_" not in k}
    ckpt = nf4_ref.to_nf4_state_dict(base, lambda mod: True) if fmt == "nf4" else tfp._fp8_checkpoint(base)[0]
    lora = {k: v for k, v in src.state_dict().items() if ".lora_" in k}
    m = type(src)(src.config, device="cpu", _host_only=True, frozen_weights=fmt)
    m.add_adapter(src.lora_rank, src.lora_rank * src.lora_scaling, target_modules=src.peft_config[src.adapter_name].target_modules)
    m.load_state_dict({**ckpt, **lora}, strict=True)
    return m


def _store_tensors(m):
    return [t for v in m._nf4_store.values() for t in v] + list(m._fp8_store.values())


def _worker(rank, world, port, family, fmt, out):
    _setup(rank, world, port)
    import test_activation_recompute as tar
    full, sh = _quantized(family, fmt), _quantized(family, fmt)
    store = _store_tensors(sh)
    store_bytes = sum(t.numel() * t.element_size() for t in store)
    alive = [weakref.ref(t) for t in store]
    del store
    assert sh.shard_frozen_weights() is sh
    freed = all(r() is None for r in alive)  # without a garbage collection: nothing waits for one to free the stacks
    assert sh.shard_frozen_weights() is sh  # a second call changes nothing, as for bf16
    rings = [r for r in (sh._sharded, sh._sharded_s) if r is not None]
    batch = (tar._qwen_batch if family == "qwen" else tar._flux_batch)("dense", seed=100 + rank)  # per-rank data
    a = tar._fused(full, family, batch)
    b = tar._fused(sh, family, batch)
    again = tar._fused(sh, family, batch)  # the second step starts from the rings as the backward left them
    res = dict(same_step=a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]),
               same_again=again[0] == b[0] and torch.equal(again[1], b[1]) and torch.equal(again[2], b[2]),
               grad_nonzero=float(a[2].norm()) > 0, loss=a[0],
               fraction=sum(r.shard.numel() * r.shard.element_size() for r in rings) / store_bytes,
               freed=freed and not sh._nf4_store and not sh._fp8_store,
               frozen_weights=sh.frozen_weights, gather=[r.gather for r in rings],
               state_keys=all("lora" in k or "transformer_blocks" not in k for k in sh.state_dict()))
    if family == "qwen":  # the no-grad forward of the sampler
        rn = tar._rn(200 + rank)
        emb = batch[0]
        kw = dict(hidden_states=rn(2, 32, 64), timestep=torch.tensor([0.5, 0.25]), encoder_hidden_states=emb["prompt_embeds"],
                  encoder_hidden_states_mask=torch.ones(2, 8, dtype=torch.int64), img_shapes=emb["img_shapes"], txt_seq_lens=[8, 8])
        with torch.no_grad():
            res["same_forward"] = torch.equal(full(**kw)[0], sh(**kw)[0])
    lora = {k: v for k, v in full.state_dict().items() if ".lora_" in k}
    missing, unexpected = sh.load_state_dict(lora, strict=False)  # a LoRA file still loads into the sharded model
    res["lora_loads"] = not unexpected
    sh.close()
    allr = [None] * world
    dist.all_gather_object(allr, res)
    if rank == 0:
        torch.save(allr, out)
    dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("fmt", ["nf4", "fp8"])
@pytest.mark.parametrize("family", ["qwen", "flux"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_codes_equal_the_unsharded_model(tmp_path, world, family, fmt):
    out = str(tmp_path / "res.pt")
    mp.spawn(_worker, args=(world, _free_port(), family, fmt, out), nprocs=world, join=True)
    res = torch.load(out)
    assert len({r["loss"] for r in res}) == world, "every rank trains on its own batch"
    for r in res:
        assert r["same_step"] and r["same_again"] and r["grad_nonzero"], r
        assert r.get("same_forward", True), r
        assert 1 / world <= r["fraction"] <= 1 / world + 0.01, r
        assert r["freed"], "the full code stacks are freed after sharding"
        assert r["frozen_weights"] == fmt and r["state_keys"] and r["lora_loads"], r
        assert r["gather"] == ["nccl"] * (1 if family == "qwen" else 2), "CPU models gather with a collective"


def _refusal_worker(rank, world, port, out):
    _setup(rank, world, port)
    from qflux_b200 import lib
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    msgs = {}
    partial = QwenImageB200(QwenB200Config(num_layers=2, num_attention_heads=2, joint_attention_dim=128), device="cpu", _host_only=True,
                            frozen_weights=("qkv_w", "out_w"))  # a checkpoint whose other block matrices are bf16
    try:
        partial.shard_frozen_weights()
    except lib.QfxError as e:
        msgs["partial"] = str(e)
    for fmt in ("nf4", "fp8"):
        sh = _quantized("qwen", fmt).shard_frozen_weights()
        try:
            sh.merge_adapter()
        except lib.QfxError as e:
            msgs["merge_" + fmt] = str(e)
    if rank == 0:
        torch.save(msgs, out)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_refusals(tmp_path):
    out = str(tmp_path / "res.pt")
    mp.spawn(_refusal_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    msgs = torch.load(out)
    assert "sharded NF4 needs every stacked block matrix NF4-resident" in msgs["partial"], msgs
    for fmt in ("nf4", "fp8"):
        assert "merge_adapter: the frozen weights are sharded" in msgs["merge_" + fmt], msgs


def test_refuses_one_rank():
    """With one rank there is nothing to shard: the unsharded ring already holds the one copy of the codes."""
    for p in (HERE, ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    from qflux_b200 import lib
    for fmt, name in (("nf4", "sharded NF4"), ("fp8", "sharded FP8")):
        m = _quantized("qwen", fmt)
        with pytest.raises(lib.QfxError, match=f"{name} needs world >= 2"):
            m.shard_frozen_weights()
        assert m._sharded is None and m.frozen_weights == fmt


# ------------------------------------------------------------------------------------------------------------------ GPU
def _gpu_case(name):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sharded_quant_check.py"), name], capture_output=True, text=True,
                       cwd=ROOT)
    print(r.stdout[-4000:], r.stderr[-4000:])
    assert r.returncode == 0, name


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", ["qwen_nf4", "qwen_fp8", "flux_nf4", "flux_fp8"])
def test_gpu(name):
    _gpu_case(name)
