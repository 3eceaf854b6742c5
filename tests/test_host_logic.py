"""Host-side logic that needs no GPU: module tree / state-dict contract, initial weights, tile heuristics, audio
helpers, synthetic batch, checkpoint loading, and the data-parallel semantics on a 2-rank gloo group."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import olmoasr_b200 as ob
from olmoasr_b200 import _core, audio, synthetic
from oracle import logmel
from oracle import model as OM


def test_state_dict_contract_and_initial_weights_match_reference():
    for train in (True, False):
        torch.manual_seed(0)
        m = (ob.model.OLMoASR if train else ob.inf_model.OLMoASR)(ob.VARIANT_TO_DIMS["tiny"])
        sd = OM.init_state_dict(OM.variant_dims("tiny"), seed=0, train=train)   # pinned to the reference in test_oracle_pin
        msd = m.state_dict()
        assert set(msd) == set(sd)
        for k in sd:
            assert msd[k].shape == sd[k].shape, k
            if train or k != "decoder.positional_embedding":   # inf_model leaves it uninitialised (inf_model.py:307)
                assert torch.equal(msd[k], sd[k]), k
        assert "decoder.mask" not in msd and m.decoder.mask.shape == (448, 448)   # non-persistent buffer
        assert m.decoder.token_embedding.weight.shape[0] == (51865 if train else 51864)
        assert m.is_multilingual is False and m.num_languages == 99
    from olmoasr_b200.model import ResidualAttentionBlock  # FSDP wrap unit must be importable (train_fsdp_timestamps.py:59-61)
    assert isinstance(m.encoder.blocks[0], ResidualAttentionBlock)


def test_parameter_counts():
    want = {"tiny": 37.18e6, "base": 71.83e6}   # SURVEY.md section 0 (train model incl. the pad row)
    for name, n in want.items():
        with torch.device("meta"):
            m = ob.model.OLMoASR(ob.VARIANT_TO_DIMS[name])
        got = sum(p.numel() for p in m.parameters())
        assert abs(got - n) / n < 2e-3, (name, got)


def test_tile_heuristics():
    _core._sm_count = lambda: 148
    assert _core._pick_block_n(48000, 1024) in (128, 256)
    assert _core._pick_block_n(100, 64) == 64
    for tiles, kb in ((32, 750), (128, 750), (1624, 224), (1, 1)):
        s = _core._pick_split_k(tiles, kb)
        assert 1 <= s <= min(8, kb)
    assert _core._pick_split_k(32, 750) > 1          # 32 output tiles cannot fill 148 SMs without split-K
    assert _core._pick_split_k(1624, 224) == 1


def test_kv_len_accepts_lengths_and_rejects_what_it_cannot_derive():
    """Key counts are derived from the dense mask by a CUDA kernel (tests/test_kernels_gpu.py); on the host only the
    argument contract is visible: integer lengths pass through, malformed masks and CPU masks raise."""
    from olmoasr_b200._lib import OasrError

    _, _, pm, lens = synthetic.text_batch(5)
    assert torch.equal(_core.kv_len_from_padding_mask(lens), lens.int())
    assert _core.kv_len_from_padding_mask(lens.int()).dtype == torch.int32
    with pytest.raises(ValueError, match="padding_mask must be"):
        _core.kv_len_from_padding_mask(pm[:, :10])             # not square
    with pytest.raises(ValueError, match="padding_mask must be"):
        _core.kv_len_from_padding_mask(pm.double())
    with pytest.raises(OasrError, match="CUDA"):
        _core.kv_len_from_padding_mask(pm.bfloat16())          # what FSDP's input cast produces: accepted (on the device)
    with pytest.raises(OasrError, match="CUDA"):
        _core.kv_len_from_padding_mask(pm)                     # no CPU path


def test_side_stream_helper_is_inert_off_cuda():
    side = _core._Side(torch.device("cpu"))
    assert not side.on
    assert side.run(lambda: 41 + 1) == 42
    side.join()


def test_audio_helpers_match_oracle():
    assert np.array_equal(audio.mel_filterbank(80), logmel.mel_filters(80))
    x = np.arange(10, dtype=np.float32)
    assert np.array_equal(audio.pad_or_trim(x, 4), logmel.pad_or_trim(x, 4))
    assert np.array_equal(audio.pad_or_trim(x, 12), logmel.pad_or_trim(x, 12))
    t = torch.arange(10.0)
    assert audio.pad_or_trim(t, 12).shape == (12,) and audio.pad_or_trim(t, 3).tolist() == [0.0, 1.0, 2.0]
    assert (audio.N_SAMPLES, audio.N_FRAMES, audio.HOP_LENGTH, audio.N_FFT) == (480000, 3000, 160, 400)
    if not torch.cuda.is_available():
        from olmoasr_b200._lib import OasrError
        with pytest.raises(OasrError):   # no silent CPU fallback
            audio.log_mel_spectrogram(np.zeros(480000, np.float32))


def test_synthetic_batch_follows_the_dataset_contract():
    ti, ty, pm, lens = synthetic.text_batch(4)
    assert ti.shape == ty.shape == (4, 448) and pm.shape == (4, 448, 448)
    for i in range(4):
        n = int(lens[i])
        assert n == 32 + (37 * i) % 192 - 1
        assert ti[i, 0] == 50257 and ti[i, 1] == 50362 and ty[i, n - 1] == 50256
        assert (ti[i, n:] == 51864).all() and (ty[i, n:] == 51864).all()
        assert torch.equal(ti[i, 1:n], ty[i, : n - 1])
        assert (pm[i, :, :n] == 0).all() and torch.isinf(pm[i, :, n:]).all()
    w = synthetic.waveforms(2, int16=True)
    assert w.dtype == torch.int16 and w.shape == (2, 480000)


def test_load_model_reads_reference_checkpoints(tmp_path):
    torch.manual_seed(1)
    dims = ob.VARIANT_TO_DIMS["tiny"]
    m = ob.model.OLMoASR(dims)
    # the reference's DDP checkpoint layout: "module."-prefixed keys, dims as the dataclass (train_timestamps.py:930-955)
    ck = {"dims": dims, "model_state_dict": {"module." + k: v for k, v in m.state_dict().items()}}
    f = tmp_path / "ddp.pt"
    torch.save(ck, f)
    m2 = ob.load_model(str(f), device="cpu")
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))
    # inference checkpoint: pad row dropped, dims as a dict (scripts/eval/gen_inf_ckpt.py:4-11)
    sd = dict(m.state_dict())
    sd["decoder.token_embedding.weight"] = sd["decoder.token_embedding.weight"][:-1]
    f2 = tmp_path / "inf.pt"
    torch.save({"dims": dict(vars(dims)), "model_state_dict": sd}, f2)
    m3 = ob.load_model(str(f2), device="cpu", inference=True, in_memory=True)
    assert m3.decoder.token_embedding.weight.shape[0] == 51864
    with pytest.raises(ValueError):
        ob.load_model("no-such-model", device="cpu")


def _small_dims():
    from olmoasr_b200.config.model_dims import ModelDimensions
    return ModelDimensions(80, 1500, 64, 1, 2, 51864, 448, 64, 1, 2)


def test_checkpoint_writer_and_gen_inf_ckpt_round_trip(tmp_path):
    """SURVEY 8(f)-4: what save_ckpt writes (train_timestamps.py:930-955, both flavours) loads back into the training model,
    converts with gen_inf_ckpt (scripts/eval/gen_inf_ckpt.py:4-11) and loads into the inference model through load_model --
    also from a model whose parameters live in slabs."""
    import olmoasr_b200 as ob
    from olmoasr_b200 import checkpoint as C
    from olmoasr_b200.model import OLMoASR

    torch.manual_seed(0)
    m = OLMoASR(_small_dims())
    m.use_slabs()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    for flavour, ddp in (("non_ddp", False), ("ddp", True)):
        path = str(tmp_path / f"latesttrain_00000007_tiny_x_{flavour}.pt")
        C.save_ckpt(path, m, opt, global_step=7, epoch=1, best_eval_wer=0.5, ddp_names=ddp)
        ck = torch.load(path, weights_only=False)
        assert set(ck) == {"global_step", "local_step", "epoch", "best_eval_wer", "model_state_dict", "optimizer_state_dict",
                           "scaler_state_dict", "scheduler_state_dict", "dims"}
        keys = list(ck["model_state_dict"])
        assert all(k.startswith("module.") for k in keys) == ddp
        sizes = {v.untyped_storage().nbytes() for v in ck["model_state_dict"].values()}
        assert max(sizes) == ck["model_state_dict"][("module." if ddp else "") + "decoder.token_embedding.weight"].numel() * 4   # no slab-sized storages
        torch.manual_seed(1)
        m2 = OLMoASR(_small_dims())
        got = C.load_ckpt(path, m2)
        assert got["global_step"] == 7 and all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))
        assert ob.load_model(path, device="cpu").state_dict().keys() == m.state_dict().keys()
        inf = C.gen_inf_ckpt(path, str(tmp_path / f"inf_{flavour}.pt"))
        ic = torch.load(inf, weights_only=False)
        assert isinstance(ic["dims"], dict) and ic["model_state_dict"]["decoder.token_embedding.weight"].shape[0] == 51864
        mi = ob.load_model(inf, device="cpu", inference=True)
        assert torch.equal(mi.decoder.token_embedding.weight, m.decoder.token_embedding.weight[:-1])
        assert torch.equal(mi.encoder.conv1.weight, m.encoder.conv1.weight)
    with pytest.raises(ValueError, match="not a training checkpoint"):
        C.gen_inf_ckpt(inf, str(tmp_path / "twice.pt"))


# ---------------------------------------------------------------------------------------------- 2-rank gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _ddp_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # per-rank shard of the synthetic batch (seeded by rank, as bench.py does) and DDP's mean-of-per-rank-means loss
    ti, ty, pm, lens = synthetic.text_batch(3, rank=rank)
    torch.manual_seed(0)
    w = torch.nn.Linear(8, 4)
    ddp = torch.nn.parallel.DistributedDataParallel(w)
    x = torch.randn(5, 8, generator=torch.Generator().manual_seed(100 + rank))
    loss = ddp(x).pow(2).mean()          # per-rank mean, like F.cross_entropy over this rank's tokens
    loss.backward()
    g = w.weight.grad.clone()
    gathered = [torch.zeros_like(g) for _ in range(world)]
    dist.all_gather(gathered, g)
    t = torch.tensor([float(rank + 1) * 10.0])
    dist.all_reduce(t, op=dist.ReduceOp.MAX)   # bench.py: max-over-ranks step time
    if rank == 0:
        torch.save({"grads": gathered, "lens": lens, "tmax": float(t)}, out)
    dist.barrier()
    dist.destroy_process_group()


def test_data_parallel_semantics_world2_gloo(tmp_path):
    out = str(tmp_path / "r0.pt")
    port = _free_port()
    mp.spawn(_ddp_worker, args=(2, port, out), nprocs=2, join=True)
    r = torch.load(out, weights_only=False)
    assert torch.allclose(r["grads"][0], r["grads"][1])           # gradients are averaged across ranks
    assert r["tmax"] == 20.0
    # ranks draw different shards
    a = synthetic.text_batch(3, rank=0)[0]
    b = synthetic.text_batch(3, rank=1)[0]
    assert not torch.equal(a, b)
    # reference arithmetic: grad of mean-of-per-rank-means == average of per-rank grads
    torch.manual_seed(0)
    w = torch.nn.Linear(8, 4)
    gs = []
    for rank in range(2):
        w.zero_grad()
        x = torch.randn(5, 8, generator=torch.Generator().manual_seed(100 + rank))
        w(x).pow(2).mean().backward()
        gs.append(w.weight.grad.clone())
    assert torch.allclose(r["grads"][0], (gs[0] + gs[1]) / 2, atol=1e-6)


class _ToyBlock(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.attn = torch.nn.Linear(6, 6)
        self.mlp = torch.nn.Linear(6, 6)
        self._param_names = [n for n, _ in self.named_parameters()]

    def forward(self, x):
        return x + self.mlp(torch.tanh(self.attn(x)))


def _blockwise_worker(rank, world, port, out, coalesce):
    from olmoasr_b200.ddp import BlockwiseGradReducer, default_buckets

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(rank)                      # different initial weights: the constructor must broadcast rank 0's
    net = torch.nn.Sequential(_ToyBlock(), _ToyBlock(), torch.nn.Linear(6, 3))
    unused = torch.nn.Parameter(torch.zeros(2))  # never receives a gradient: finish() must still terminate
    net.register_parameter("unused", unused)
    red = BlockwiseGradReducer(net, coalesce=coalesce)
    assert [len(b) for b in default_buckets(net)] == [4, 4, 3]
    results = []
    for it in range(2):                          # two steps: the reducer re-arms itself
        net.zero_grad(set_to_none=True)
        x = torch.randn(5, 6, generator=torch.Generator().manual_seed(100 * it + rank))
        net(x).pow(2).mean().backward()
        inv = red.finish()
        results.append([p.grad.clone() * inv for p in net.parameters() if p.grad is not None])
    w0 = [p.detach().clone() for p in net.parameters()]
    if rank == 0:
        torch.save({"grads": results, "weights": w0}, out)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("coalesce", [True, False])
def test_blockwise_grad_reducer_matches_ddp_averaging_world2_gloo(tmp_path, coalesce):
    out = str(tmp_path / "r0.pt")
    mp.spawn(_blockwise_worker, args=(2, _free_port(), out, coalesce), nprocs=2, join=True)
    r = torch.load(out, weights_only=False)
    # reference arithmetic on one process: average of the per-rank gradients, starting from rank 0's weights
    torch.manual_seed(0)
    net = torch.nn.Sequential(_ToyBlock(), _ToyBlock(), torch.nn.Linear(6, 3))
    net.register_parameter("unused", torch.nn.Parameter(torch.zeros(2)))
    for a, b in zip(net.parameters(), r["weights"]):
        assert torch.equal(a.detach(), b)
    for it in range(2):
        per_rank = []
        for rank in range(2):
            net.zero_grad(set_to_none=True)
            x = torch.randn(5, 6, generator=torch.Generator().manual_seed(100 * it + rank))
            net(x).pow(2).mean().backward()
            per_rank.append([p.grad.clone() for p in net.parameters() if p.grad is not None])
        for got, g0, g1 in zip(r["grads"][it], per_rank[0], per_rank[1]):
            assert torch.allclose(got, (g0 + g1) / 2, atol=1e-6)


# ---------------------------------------------------------------------------------------------- parameter slabs (host logic)

def test_slab_layout_keeps_the_state_dict_and_gives_fused_views():
    from olmoasr_b200.model import OLMoASR

    torch.manual_seed(0)
    m = OLMoASR(_small_dims())
    before = {k: v.clone() for k, v in m.state_dict().items()}
    n_params = sum(p.numel() for p in m.parameters())
    sl = m.use_slabs()
    after = m.state_dict()
    assert list(after) == list(before) and all(torch.equal(after[k], before[k]) for k in before)   # names, order, values
    assert n_params <= sl.numel <= n_params + 64 * 64                     # only the zero gaps of the bias-less key projections
    assert all(p.data_ptr() == sl.P.data_ptr() + 4 * sl.offset[id(p)] for p in m.parameters())
    assert all(p.grad.data_ptr() == sl.G.data_ptr() + 4 * sl.offset[id(p)] for p in m.parameters())
    for blk in list(m.encoder.blocks) + list(m.decoder.blocks):
        for a in (blk.attn, blk.cross_attn):
            if a is None:
                continue
            w, b = a.fused_qkv()
            d = a.query.weight.shape[0]
            assert w.shape == (3 * d, d) and w.dtype == torch.bfloat16 and b.shape == (3 * d,) and b.dtype == torch.float32
            assert torch.equal(b[:d], a.query.bias) and torch.equal(b[2 * d:], a.value.bias) and float(b[d:2 * d].abs().max()) == 0
            assert w.data_ptr() == sl.S.data_ptr() + 2 * sl.offset[id(a.query.weight)]
            wk, bk = a.fused_kv()
            assert wk.shape == (2 * d, d) and wk.data_ptr() == sl.S.data_ptr() + 2 * sl.offset[id(a.key.weight)]
    # layout order == backward completion order: decoder first, conv stem last
    assert sl.offset[id(m.decoder.ln.weight)] == 0
    assert sl.offset[id(m.encoder.conv1.bias)] == max(sl.offset.values())
    assert sl.offset[id(m.decoder.blocks[1].mlp_ln.weight)] < sl.offset[id(m.decoder.blocks[0].mlp_ln.weight)]
    # load_state_dict writes through the views and bumps the versions the shadow sync keys on
    sig = sl._signature()
    m.load_state_dict({k: v + 1.0 if v.is_floating_point() else v for k, v in before.items()})
    assert sl._signature() != sig and torch.equal(sl.span("P", m.decoder.ln.weight, 64), before["decoder.ln.weight"] + 1.0)
    # zero_grad is one memset and re-attaches dropped views
    m.decoder.ln.weight.grad = None
    sl.G.fill_(3.0)
    sl.zero_grad()
    assert float(sl.G.abs().max()) == 0 and m.decoder.ln.weight.grad.data_ptr() == sl.G.data_ptr()
    # grad_units partition the layout in order (what SlabGradSync cuts into all-reduce segments)
    order = {pid: i for i, pid in enumerate(sl.layout_order)}
    nxt = 0
    for ps, mod in m.grad_units():
        idx = sorted(order[id(p)] for p in ps)
        assert idx == list(range(nxt, nxt + len(ps)))
        nxt += len(ps)
    assert nxt == len(order)
    with pytest.raises(ValueError, match="every trainable parameter"):
        from olmoasr_b200.slab import ParamSlabs
        ParamSlabs(torch.nn.Linear(4, 4), layout=[])


class _ToySlabModel(torch.nn.Module):
    """Two 'blocks' + a head with the grad_units / _bwd_done_cb protocol of OLMoASRBase (host logic only)."""

    def __init__(self):
        super().__init__()
        self.b0, self.b1, self.head = torch.nn.Linear(64, 64), torch.nn.Linear(64, 64), torch.nn.Linear(64, 64)
        for mod in (self.b0, self.b1, self.head):
            mod._bwd_done_cb = None

    def forward(self, x):
        return self.head(torch.tanh(self.b1(torch.tanh(self.b0(x)))))

    def grad_units(self):   # backward order: head, b1, b0
        return [(list(self.head.parameters()), self.head), (list(self.b1.parameters()), self.b1), (list(self.b0.parameters()), self.b0)]


def _slab_sync_worker(rank, world, port, out):
    from olmoasr_b200.ddp import SlabGradSync
    from olmoasr_b200.slab import ParamSlabs

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(rank)                       # different initial weights: the constructor must broadcast rank 0's
    net = _ToySlabModel()
    layout = [p for ps, _ in net.grad_units() for p in ps]
    slabs = ParamSlabs(net, layout, shadows=False)
    sync = SlabGradSync(net, slabs, bucket_bytes=1, tail_bucket_bytes=1)      # every unit its own segment
    assert len(sync.segments) == 3 and sync.segments[0][0] == 0 and sync.segments[-1][1] == slabs.numel
    assert all(a[1] == b[0] for a, b in zip(sync.segments, sync.segments[1:]))
    launched_early = []
    results = []
    for it in range(3):
        slabs.zero_grad()
        x = torch.randn(5, 64, generator=torch.Generator().manual_seed(100 * it + rank))
        loss = net(x).pow(2).mean()
        if it == 2:                                # gradient accumulation: first micro-batch inside no_sync()
            with sync.no_sync():
                loss.backward()
                for mod in (net.head, net.b1, net.b0):
                    mod._bwd_done_cb()
                assert not sync._works
            x = torch.randn(5, 64, generator=torch.Generator().manual_seed(999 + rank))
            loss = net(x).pow(2).mean()
        loss.backward()                            # autograd accumulates into the slab views
        for mod in (net.head, net.b1):             # the fused backward fires these as it goes; b0's never fires here
            mod._bwd_done_cb()
        launched_early.append(list(sync._launched))
        inv = sync.finish()                        # launches the segment nobody triggered, waits, re-arms
        results.append((slabs.G * inv).clone())
    if rank == 0:
        torch.save({"grads": results, "weights": slabs.P.clone(), "early": launched_early, "offsets": [slabs.offset[id(p)] for p in layout]}, out)
    dist.barrier()
    dist.destroy_process_group()


def test_slab_grad_sync_matches_ddp_averaging_world2_gloo(tmp_path):
    out = str(tmp_path / "r0.pt")
    mp.spawn(_slab_sync_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    r = torch.load(out, weights_only=False)
    assert r["early"][0] == [True, True, False]
    torch.manual_seed(0)
    net = _ToySlabModel()
    layout = [p for ps, _ in net.grad_units() for p in ps]
    flat_w = torch.cat([p.detach().reshape(-1) for p in layout])
    assert torch.equal(r["weights"][: flat_w.numel()], flat_w)          # rank 0's weights everywhere (sizes are 64-multiples: no gaps)

    def per_rank_grads(seed_fn):
        gs = []
        for rank in range(2):
            net.zero_grad(set_to_none=True)
            for seed in seed_fn(rank):
                x = torch.randn(5, 64, generator=torch.Generator().manual_seed(seed))
                net(x).pow(2).mean().backward()
            gs.append(torch.cat([p.grad.reshape(-1) for p in layout]))
        return (gs[0] + gs[1]) / 2

    for it in range(2):
        assert torch.allclose(r["grads"][it], per_rank_grads(lambda rank: [100 * it + rank]), atol=1e-6)
    assert torch.allclose(r["grads"][2], per_rank_grads(lambda rank: [200 + rank, 999 + rank]), atol=1e-6)   # accumulated, synced once
