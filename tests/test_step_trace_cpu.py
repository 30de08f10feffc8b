"""The launch sequence of one DiT step, pinned without a GPU.

Both drop-ins (miniFLUX and the SD3 MMDiT) are built on the CPU at a small synthetic size, and `_forward_eager` runs with the
launching functions of `pyramid_flow_b200.ops` replaced by recorders.  The sequence-parallel exchanges are replaced by
recording fakes, so the CFG x sequence-parallel branches, which otherwise run only on several GPUs, are covered too.
Every launch is recorded with all its arguments (defaults applied); a tensor is described by the ordinal of its storage in
order of first use, its storage offset, shape, stride and dtype, so aliasing into shared buffers is part of the trace.
The host schedule builders are the real ones.  The result must equal tests/golden/dit_step_trace.pt case by case.

    python tests/test_step_trace_cpu.py --write      re-records the fixture
"""
import inspect
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from pyramid_flow_b200 import _lib, ops, sp  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "dit_step_trace.pt"
RECORDED = ("gemm", "gemm_fp8", "ln_modulate", "ln_modulate_fp8", "quantize_rows_fp8", "small_linear", "timestep_embedding",
            "patchify", "unpatchify", "attn_fwd")
TEXT_LEN = 16
# two clips: 2 x 8 x 8 and 1 x 16 x 16 tokens; S = 16 + 128 + 256 = 400, so the trimmed last single block starts at row 128
CLIPS = ((2, 16, 2, 16, 16), (2, 16, 1, 32, 32))
FAKE_PTRS = (0x7f0000000000, 0x7f1000000000, 0x7f2000000000, 0x7f3000000000)


class Trace:
    def __init__(self):
        self.events = []
        self._storages = {}
        self._keep = []          # every described tensor stays alive, so no storage address is reused within a trace

    def tensor(self, t):
        key = t.untyped_storage().data_ptr()
        if key not in self._storages:
            self._storages[key] = len(self._storages)
            self._keep.append(t)
        return ("tensor", self._storages[key], t.storage_offset(), tuple(t.shape), tuple(t.stride()), str(t.dtype))

    def describe(self, x):
        if isinstance(x, torch.Tensor):
            return self.tensor(x)
        if isinstance(x, ops.PairSchedule):
            return ("PairSchedule", self.tensor(x.sched), self.tensor(x.mask_index), self.tensor(x.mask_bits),
                    self.describe(x.group3))
        if isinstance(x, sp.ParallelLayout):
            return ("layout", x.world, x.rank, x.cfg_ways, x.sp, x.cfg_rank, x.sp_rank)
        if isinstance(x, (list, tuple)):
            return tuple(self.describe(v) for v in x)
        if isinstance(x, dict):
            return {k: self.describe(v) for k, v in x.items()}
        if x is None or isinstance(x, (bool, int, float, str)):
            return x
        if isinstance(x, FakeBuffer):
            return ("buffer", x.name)
        raise TypeError(f"no trace description for {type(x)}")

    def record(self, name, args):
        self.events.append((name, self.describe(args)))


def _bind(fn, args, kw):
    ba = inspect.signature(fn).bind(*args, **kw)
    ba.apply_defaults()
    return dict(ba.arguments)


def _recorder(trace, name, orig):
    def gemm_args(args, kw):
        # the launch's full descriptor arguments: the positional operands of the entry, then _gemm_desc's keywords
        a = _bind(orig, args, kw)
        extra = a.pop("kw")
        desc = _bind(ops._gemm_desc, (a["a8" if "a8" in a else "a"], a["w8" if "w8" in a else "w"], a["bias"],
                                      a["epilogue"]), extra)
        return {**a, **desc}

    def rec(*args, **kw):
        trace.record(name, gemm_args(args, kw) if name in ("gemm", "gemm_fp8") else _bind(orig, args, kw))
        if name == "timestep_embedding":
            return torch.zeros(args[0].shape[0], args[1], dtype=torch.float32)
        return None

    return rec


class FakeBuffer:
    def __init__(self, name, ptrs):
        self.name, self.ptrs = name, list(ptrs)


class FakePeerExchange:
    """Stands in for sp.PeerExchange: CPU-backed views, fixed fake peer pointers and offsets, recorded collective pieces."""

    def __init__(self, trace, lay, args):
        self.trace, self.lay = trace, lay
        trace.record("ensure_peer_exchange", args)
        _, _, seq, last, hp, ldc, head_cols, vel_bytes = args
        self.hg, self.ldc, self.head_cols = hp // lay.sp, ldc, head_cols
        self.off_qkv, self.off_cat, self.off_head, self.w_off_vel = 256, 1 << 20, 2 << 20, 256
        self.vel_bytes = (vel_bytes + 255) // 256 * 256
        self.sp_buf = FakeBuffer("sp", FAKE_PTRS[:lay.sp])
        self.world_buf = FakeBuffer("world", FAKE_PTRS[:lay.world])
        self._qkv = torch.zeros(3, self.hg, seq, 64, dtype=torch.bfloat16)
        self._cat = torch.zeros(1, seq // lay.sp, ldc, dtype=torch.bfloat16)
        self._head = torch.zeros(1, last, head_cols, dtype=torch.float32)
        self._vel = torch.zeros(lay.cfg_ways, self.vel_bytes, dtype=torch.uint8)

    def qkv(self, seq):
        return self._qkv[:, :, :seq]

    def cat(self, sl):
        return self._cat[:, :sl]

    def head(self, n_last):
        return self._head[:, :n_last]

    def vel(self, shape, dtype):
        n = 1
        for s in shape[1:]:
            n *= int(s)
        es = torch.empty(0, dtype=dtype).element_size()
        return self._vel[:, :n * es].view(dtype).view(self.lay.cfg_ways, *shape[1:])

    def barrier_sp(self):
        self.trace.record("barrier_sp", ())

    def barrier_world(self):
        self.trace.record("barrier_world", ())

    def bcast(self, buf, src, dst_offset):
        self.trace.record("bcast", (buf, src, dst_offset))


def _flux(precision):
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    # 3 heads: padded to 4 under sequence parallelism of degree 2 or 4
    kw = dict(num_layers=2, num_single_layers=2, num_attention_heads=3, attention_head_dim=64, in_channels=64,
              joint_attention_dim=128, pooled_projection_dim=64)
    params = FO.synthetic_flux_params(FO.FluxConfig(**kw), seed=0)
    return B200FluxTransformer(FluxConfigB200(**kw), params, device="cpu", gemm_precision=precision)


def _mmdit(precision):
    from oracle import mmdit_oracle as MO
    from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200
    kw = dict(num_layers=3, num_attention_heads=4, attention_head_dim=64, in_channels=16, joint_attention_dim=128,
              pooled_projection_dim=64, pos_embed_max_size=16)
    params = MO.synthetic_mmdit_params(MO.MMDiTConfig(sample_size=32, **kw), seed=0)
    return B200MMDiT(MMDiTConfigB200(**kw), params, device="cpu", gemm_precision=precision)


# name -> (model, precision, trim_last_block, world, rank, exchange); world 1 = one GPU
CASES = {
    "flux_bf16": ("flux", "bf16", True, 1, 0, None),
    "flux_bf16_untrimmed": ("flux", "bf16", False, 1, 0, None),
    "flux_fp8": ("flux", "fp8", True, 1, 0, None),
    "flux_fp8_untrimmed": ("flux", "fp8", False, 1, 0, None),
    "mmdit_bf16": ("mmdit", "bf16", True, 1, 0, None),
    "mmdit_fp8": ("mmdit", "fp8", True, 1, 0, None),
    "flux_peer_cfg2sp1_r1": ("flux", "bf16", True, 2, 1, "peer"),
    "flux_peer_cfg2sp2_r0": ("flux", "bf16", True, 4, 0, "peer"),
    "flux_peer_cfg2sp2_r1": ("flux", "bf16", True, 4, 1, "peer"),
    "flux_peer_cfg2sp2_r3": ("flux", "bf16", True, 4, 3, "peer"),
    "flux_nccl_cfg2sp1_r0": ("flux", "bf16", True, 2, 0, "nccl"),
    "flux_nccl_cfg2sp2_r0": ("flux", "bf16", True, 4, 0, "nccl"),
    "flux_nccl_cfg2sp2_r3": ("flux", "bf16", True, 4, 3, "nccl"),
    "mmdit_peer_cfg2sp1_r0": ("mmdit", "bf16", True, 2, 0, "peer"),
    "mmdit_peer_cfg2sp2_r0": ("mmdit", "bf16", True, 4, 0, "peer"),
    "mmdit_peer_cfg2sp2_r1": ("mmdit", "bf16", True, 4, 1, "peer"),
    "mmdit_peer_cfg2sp2_r2": ("mmdit", "bf16", True, 4, 2, "peer"),
}


def _inputs(model):
    g = torch.Generator().manual_seed(0)
    cfg = model.config
    clips = [torch.randn(*s, generator=g) for s in CLIPS]
    t = torch.tensor([0.75, 0.75]).bfloat16().float()
    enc = torch.randn(2, TEXT_LEN, cfg.joint_attention_dim, generator=g)
    mask = torch.ones(2, TEXT_LEN, dtype=torch.long)
    mask[0, 11:] = 0
    pooled = torch.randn(2, cfg.pooled_projection_dim, generator=g)
    return clips, t, enc, mask, pooled


def run_case(name, mp):
    kind, precision, trim, world, rank, exchange = CASES[name]
    trace = Trace()
    model = _flux(precision) if kind == "flux" else _mmdit(precision)
    for fn in RECORDED:
        mp.setattr(ops, fn, _recorder(trace, fn, getattr(ops, fn)))
    mp.setattr(_lib, "require_device", lambda: None)
    if kind == "flux":
        model.trim_last_block = trim
    if world > 1:
        lay = sp.make_layout(world, rank, create_groups=False)
        fake = {}

        def ensure(owner, *args):
            if "px" not in fake:
                fake["px"] = FakePeerExchange(trace, lay, ("owner", *args))
            else:
                trace.record("ensure_peer_exchange", ("owner", *args))
            return fake["px"]

        def begin(q, k, v, lay_):
            trace.record("heads_to_sequence_qkv_begin", (q, k, v, lay_))
            return ("pending", q.shape)

        def end(handle):
            trace.record("heads_to_sequence_qkv_end", ())
            hp, sl, hd = handle[1]
            return tuple(torch.zeros(hp // lay.sp, sl * lay.sp, hd, dtype=torch.bfloat16) for _ in range(3))

        def seq_to_heads(o, lay_):
            trace.record("sequence_to_heads", (o, lay_))
            return torch.zeros(o.shape[0] // lay.sp, lay.sp * o.shape[1], dtype=o.dtype)

        mp.setattr(sp, "ensure_peer_exchange", ensure)
        mp.setattr(sp, "heads_to_sequence_qkv_begin", begin)
        mp.setattr(sp, "heads_to_sequence_qkv_end", end)
        mp.setattr(sp, "sequence_to_heads", seq_to_heads)
        mp.setattr(torch.distributed, "all_reduce", lambda t, group=None: trace.record("all_reduce", (t, group)))
        mp.setattr(torch.distributed, "all_gather_into_tensor",
                   lambda out, x, group=None: trace.record("all_gather_into_tensor", (out, x, group)))
        if kind == "flux":
            model.set_parallel_layout(lay, exchange)
        else:
            model.set_parallel_layout(lay)
    clips, t, enc, mask, pooled = _inputs(model)
    out = model._forward_eager(clips, t, enc, mask, pooled)
    trace.record("return", tuple(out))
    return trace.events


@pytest.fixture
def keep_attn_option():
    # set_parallel_layout pins the process to one attention kernel; later tests in this process get the option back
    saved = _lib.get_option(_lib.PF_OPT_ATTN_TRIPLE_KERNEL)
    yield
    _lib.set_option(_lib.PF_OPT_ATTN_TRIPLE_KERNEL, saved)


@pytest.mark.parametrize("name", sorted(CASES))
def test_step_launch_sequence_matches_the_recorded_trace(name, monkeypatch, keep_attn_option):
    want = torch.load(GOLDEN, weights_only=True)[name]
    got = run_case(name, monkeypatch)
    assert len(got) == len(want), (len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"launch {i}: {g[0]} differs\n got  {g}\n want {w}"


def _write():
    saved = _lib.get_option(_lib.PF_OPT_ATTN_TRIPLE_KERNEL)
    traces = {}
    for name in sorted(CASES):
        with pytest.MonkeyPatch.context() as mp:
            traces[name] = run_case(name, mp)
        print(f"{name}: {len(traces[name])} launches")
    _lib.set_option(_lib.PF_OPT_ATTN_TRIPLE_KERNEL, saved)
    torch.save(traces, GOLDEN)


if __name__ == "__main__":
    if sys.argv[1:] != ["--write"]:
        sys.exit(__doc__)
    _write()
