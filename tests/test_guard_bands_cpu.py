"""Guard mode of the launch checker (`Shadow(guard=True)`, tests/launch_check.py), without a GPU.

  * the tiny programs of test_launch_check_cpu.py run with every launch relocated between poisoned
    guard bands, reproduce the same golden vectors, and every launch is guarded;
  * relocation keeps each storage's address modulo 4096, every view's offset, shape and strides,
    and the aliasing of the arguments (`residual is out`, two views of one arena), and poisons
    exactly the bytes no argument views;
  * mutations applied to the relocated buffers after the fake write -- an element past the end of
    an output's storage, one before its start, a byte in an unviewed gap of an arena, an output
    recomputed from the element after its input view, a returned tensor written one row too long --
    each fail with a message that names the region.

Every out-of-bounds access simulated here is a write by a fake kernel on host memory.
"""
import pytest
import torch

import launch_check as lc
import test_launch_check_cpu as lcc
from audio_diffusion_pytorch_b200 import ops
from test_launch_check_cpu import cpu_launches, tiny_nets  # noqa: F401  (fixtures)

F64 = torch.float64


class _GuardedShadow(lc.Shadow):
    """Shadow with guard=True; every instance is kept so the test can read its counts."""
    made = []

    def __init__(self, **kw):
        super().__init__(guard=True, **kw)
        _GuardedShadow.made.append(self)


@pytest.fixture
def guarded(monkeypatch):
    _GuardedShadow.made = []
    monkeypatch.setattr(lc, "Shadow", _GuardedShadow)
    yield _GuardedShadow.made
    assert _GuardedShadow.made, "no Shadow was made"
    for sh in _GuardedShadow.made:
        assert sh.n_guarded == sh.n_launch > 0, sh.table()


# ------------------------------------------------------------------------------ programs
def test_tiny_program_guarded(cpu_launches, guarded, oracle_port, golden_dir):
    lcc.test_tiny_program_vs_golden(None, oracle_port, golden_dir)


def test_tiny_sampling_program_guarded(cpu_launches, guarded, oracle_port, golden_dir):
    lcc.test_tiny_sampling_program_vs_golden(None, oracle_port, golden_dir)


def test_text_cfg_program_guarded(cpu_launches, guarded, oracle_port, golden_dir):
    lcc.test_text_cfg_program_vs_golden(None, oracle_port, golden_dir)


def test_inpainter_program_guarded(cpu_launches, guarded, oracle_port, golden_dir, monkeypatch):
    lcc.test_inpainter_program_vs_golden(None, oracle_port, golden_dir, monkeypatch)


def test_autoregressive_program_guarded(cpu_launches, guarded, oracle_port, golden_dir, monkeypatch):
    lcc.test_autoregressive_program_vs_golden(None, oracle_port, golden_dir, monkeypatch)


def test_unfused_program_guarded(cpu_launches, guarded, oracle_port):
    lcc.test_unfused_program_probes(None, oracle_port)


@pytest.mark.parametrize("kind", ["gn_stats", "sampler_step"])
def test_direct_launch_guarded(cpu_launches, guarded, kind):
    lcc.test_direct_launch_probe(None, kind)


# ---------------------------------------------------------------------------- relocation
def _raise(msg):
    raise lc.CheckError(msg)


def test_relocation_keeps_residues_strides_and_aliasing():
    arena = torch.randn(4096 + 37)
    x = arena[5:5 + 600].view(2, 300)                  # two views of one arena, a gap between them
    v = arena[1000:1000 + 2 * 300 * 2].view(2, 300, 2)[..., 1]     # strided: every other element
    out = torch.randn(3, 40, 16, dtype=torch.bfloat16)
    col = out[..., 8:]                                 # a column view of `out`
    stats = torch.zeros(3, 4, 2, dtype=F64)
    idx = torch.arange(7, dtype=torch.int32)
    args = {"x": x, "v": v, "out": out, "residual": out, "col": col, "gn": (stats, idx, 4, 1e-5), "n": 3}
    g = lc.Guards()
    r = g.relocate(args)
    assert r["residual"] is r["out"] and r["n"] == 3 and r["gn"][2:] == (4, 1e-5)
    assert lc._key(r["x"]) == lc._key(r["v"]) != lc._key(x)
    assert lc._key(r["col"]) == lc._key(r["out"])
    for name, orig, moved in (("x", x, r["x"]), ("v", v, r["v"]), ("out", out, r["out"]), ("col", col, r["col"]),
                              ("stats", stats, r["gn"][0]), ("idx", idx, r["gn"][1])):
        assert moved.data_ptr() % lc.GUARD_ALIGN == orig.data_ptr() % lc.GUARD_ALIGN, name
        assert moved.untyped_storage().data_ptr() != orig.untyped_storage().data_ptr(), name
        assert (moved.shape, moved.stride(), moved.dtype) == (orig.shape, orig.stride(), orig.dtype), name
        assert torch.equal(lc._bits(moved), lc._bits(orig)), name
    copy, _ = g.items[lc._key(x)]
    viewed = copy.mask.bool()
    assert int(viewed.sum()) == (600 + 600) * 4        # x and every other element of the strided view
    assert bool((copy.copy[~viewed] == lc.POISON_FLOAT).all())
    assert copy.off >= lc.GUARD_BYTES and copy.buf.numel() - copy.off - copy.n >= lc.GUARD_BYTES
    assert float(r["v"].reshape(-1)[0]) == float(v.reshape(-1)[0])
    gap = torch.empty(0).set_(r["x"].untyped_storage(), r["x"].storage_offset() + 600, (1,), (1,))
    assert float(gap[0]) == pytest.approx(3.39e38, rel=1e-2)       # 0x7F7F7F7F
    int_copy, _ = g.items[lc._key(idx)]
    assert int_copy.poison == 0 and bool((int_copy.buf[:int_copy.off] == 0).all())
    g.check(_raise)              # nothing written: every guard intact
    r["out"].zero_()
    g.copy_back()
    assert not out.any() and stats.eq(0).all()


def test_allocated_results_sit_between_guards():
    g = lc.Guards()
    torch_ = g.torch_proxy()
    y = torch_.empty(3, 50, dtype=torch.float32, device="cpu")
    z = torch_.zeros_like(y)
    assert y.shape == (3, 50) and y.is_contiguous() and bool((lc._bits(y) == 0x7F7F7F7F).all())
    assert not z.any() and torch_.float32 is torch.float32 and torch_.arange(3).tolist() == [0, 1, 2]
    y.fill_(1.0)
    g.check(_raise)
    torch.empty(0).set_(z.untyped_storage(), z.storage_offset() + z.numel(), (1,), (1,)).fill_(2.0)
    with pytest.raises(lc.CheckError, match="`result` damaged past the end: 1 bytes past the end of the storage, "
                                             "1 bytes"):
        g.check(_raise)


# ----------------------------------------------------------------------------- mutations
def _copy_span(run_view, pre_view):
    """(element index of the copy's first element in the relocated buffer, elements in the copy)
    of the storage run_view lies in: pre_view is the same view on the snapshot, whose storage has
    the original's size."""
    es = run_view.element_size()
    return run_view.storage_offset() - pre_view.storage_offset(), pre_view.untyped_storage().nbytes() // es


def _at(view, index):
    """One element of view's buffer at element index `index` (anywhere in the buffer)."""
    return torch.empty(0, dtype=view.dtype).set_(view.untyped_storage(), index, (1,), (1,))


def _first_val(outs):
    return next(o for o in outs if isinstance(o, lc.Val))


def m_past_end(post, outs, pre):
    """One element written just past the end of the first output's storage."""
    o = _first_val(outs)
    start, n = _copy_span(o.view(post), o.view(pre))
    _at(o.view(post), start + n).fill_(1)


def m_before_start(post, outs, pre):
    """One element written just before the start of the first output's storage."""
    o = _first_val(outs)
    start, _ = _copy_span(o.view(post), o.view(pre))
    _at(o.view(post), start - 1).fill_(1)


def m_gap_byte(post, outs, pre):
    """One byte written into the first byte of the output's storage that no argument views."""
    o = _first_val(outs)
    v = o.view(post)
    start, n = _copy_span(v, o.view(pre))
    start *= v.element_size()
    n *= v.element_size()
    viewed = torch.zeros(n, dtype=torch.bool)
    for t in lc._tensors(list(post.values())):
        if lc._key(t) == lc._key(v):
            lo, hi = lc._extent(t)
            viewed[lo - start:hi - start] = True
    free = (~viewed).nonzero()
    if not free.numel():
        return False
    _at(lc._bits(v).view(torch.uint8), start + int(free[0, 0])).fill_(1)


def m_over_read(post, outs, pre):
    """sampler_step: the last element of x_next computed from the element after x's view."""
    x, v, x_next = post["x"], post["v"], post["x_next"]
    assert x.is_contiguous()
    after = _at(x, x.storage_offset() + x.numel()).to(F64)
    a0, b0, a1, b1 = pre["ab"].to(F64).tolist()
    vl = v.reshape(-1)[-1].to(F64)
    x_next.view(-1)[-1] = a1 * (a0 * after - b0 * vl) + b1 * (b0 * after + a0 * vl)


def m_result_row_too_long(post, outs, pre):
    """A returned tensor [rows, n] written one row too long (row `rows` is past its end)."""
    o = _first_val(outs)
    out = o.view(post)
    assert out.is_contiguous()
    torch.empty(0, dtype=out.dtype).set_(out.untyped_storage(), out.storage_offset(),
                                         (out.shape[0] + 1, out.shape[1]), (out.shape[1], 1)).fill_(0.5)


def _arena_step():
    """sampler_step on three views of one arena, with gaps between them and after the last."""
    g = torch.Generator().manual_seed(3)
    arena = torch.randn(3 * 1024, generator=g)
    x, v, x_next = (arena[i * 1024:i * 1024 + 1000].view(2, 2, 250) for i in range(3))
    ops.sampler_step(x, v, torch.tensor([0.8, 0.6, 0.9, 0.43589]), x_next)
    return arena


def _to_flat():
    g = torch.Generator().manual_seed(4)
    return ops.to_flat(torch.randn(2, 4, 9, generator=g), torch.randn(4, 16, generator=g), 4, 6)


def _fir_resample():
    g = torch.Generator().manual_seed(6)
    return ops.fir_resample(torch.randn(3, 100, generator=g), torch.randn(2, 8, generator=g), 1, 2, 4, 200)


GUARD_MUTANTS = [  # (mutation, kind, program, what the message must say)
    (m_past_end, "conv_gemm", "v", "guard: `out` damaged past the end: 1 bytes past the end of the storage"),
    (m_past_end, "sampler_step", "arena", "guard: `x_next` damaged past the end"),
    (m_before_start, "stem_out", "v", "guard: `v_out` damaged before the start: 1 bytes before the start"),
    (m_before_start, "sampler_step", "arena", "guard: `x` damaged before the start"),
    (m_gap_byte, "sampler_step", "arena", "guard: `x` damaged in an unviewed gap: storage byte 4000, 1 bytes"),
    (m_over_read, "sampler_step", "arena", "x_next[1, 1, 249]: got 3.3"),
    (m_result_row_too_long, "to_flat", "to_flat", "guard: `out` damaged past the end: 1 bytes past the end"),
    (m_result_row_too_long, "fir_resample", "fir_resample", "guard: `_result` damaged past the end"),
]


@pytest.mark.parametrize("mutation,kind,program,message", GUARD_MUTANTS,
                         ids=[f"{m.__name__[2:]}-{k}" for m, k, _, _ in GUARD_MUTANTS])
def test_guard_mutation_is_caught(cpu_launches, tiny_nets, mutation, kind, program, message):
    g = torch.Generator().manual_seed(11)
    with torch.no_grad(), lc.Shadow(fake=True, guard=True, mutate=(kind, mutation)) as sh:
        with pytest.raises(lc.CheckError) as err:
            if program == "v":
                tiny_nets["fused"](torch.randn(2, 2, 4096, generator=g), torch.rand(2, generator=g))
            else:
                {"arena": _arena_step, "to_flat": _to_flat, "fir_resample": _fir_resample}[program]()
    assert sh.mutate is None, f"{mutation.__name__} never applied to a {kind} launch"
    assert f"): {kind}: " in str(err.value) and message in str(err.value), str(err.value)
    print(f"caught {mutation.__name__} in {kind}: {err.value}")


@pytest.mark.parametrize("program", ["arena", "to_flat", "fir_resample"])
def test_direct_programs_pass_guarded(cpu_launches, program):
    """The mutation tests' direct launches pass unmutated, and return what an unguarded run does."""
    fn = {"arena": _arena_step, "to_flat": _to_flat, "fir_resample": _fir_resample}[program]
    with lc.Shadow(fake=True) as plain:
        want = fn()
    with lc.Shadow(fake=True, guard=True) as sh:
        got = fn()
    assert sh.n_guarded == sh.n_launch == plain.n_launch == 1
    assert torch.equal(got, want)
    if program == "arena":                 # the gaps between the views hold what they held
        assert torch.equal(got[1000:1024], torch.randn(3 * 1024, generator=torch.Generator().manual_seed(3))[1000:1024])
    else:
        assert got.untyped_storage().nbytes() == got.numel() * 4      # a plain copy, not a view of a guard buffer
