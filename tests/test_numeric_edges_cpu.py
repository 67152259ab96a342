"""The checks of tests/test_numeric_edges_gpu.py can fail: run on the CPU in the launch checker's
fake mode (each launch writes its fp64 restatement), with a mutation standing in for a kernel that
gets the numerics wrong.

  a. statistics: the slots replaced by a single-pass fp32 sequential sum over the whole group.
     The launch checker's own statistics bound sees it at the producer; with that bound switched
     off, the consumer comparison (GroupNorm from a two-pass fp64 variance of the input) still
     fails the R = 256 group -- the launch checker's consumer checks, which start from the
     statistics the consumer was given, pass.
  c. attention: an online softmax over 128-key tiles that drops the rescale of what earlier tiles
     accumulated (alpha = 1) fails the case whose row maximum arrives in the last key tile, and
     is exact where the maximum never moves (all-equal logits)."""
import math

import pytest
import torch

import launch_check as lc
import test_numeric_edges_gpu as ne

T_CPU = 1 << 16                 # 2^16 rows x 32 channels per group: 2M-term sums, as on the GPU at 2^16


class _StatsUnbounded(lc.Shadow):
    """The launch checker with its statistics bound off: only what the consumer comparison sees."""

    def _check_stats(self, *args):
        pass


def test_statistics_consumer_comparison_passes_exact_statistics():
    rows = ne.stats_case("gn_stats", ne.KINDS, lambda: lc.Shadow(fake=True, probe=True), T=T_CPU, dev="cpu")
    assert max(v for r in rows for v in r[6].values()) <= 1.0
    r256 = next(r for r in rows if r[1] == "R256")
    assert 200 < r256[2] < 300, r256                         # the R the rounded tensor has


def test_fp32_sequential_statistics_fail_the_producer_bound():
    with pytest.raises(lc.CheckError, match="gn_stats: stats"):
        ne.stats_case("gn_stats", ne.KINDS, lambda: lc.Shadow(fake=True, mutate=("gn_stats", ne.m_fp32_sequential)),
                      T=T_CPU, dev="cpu")


def test_fp32_sequential_statistics_fail_the_consumer_comparison():
    with pytest.raises(lc.CheckError) as e:
        ne.stats_case("gn_stats", ne.KINDS,
                      lambda: _StatsUnbounded(fake=True, mutate=("gn_stats", ne.m_fp32_sequential)),
                      T=T_CPU, dev="cpu")
    msg = str(e.value)
    assert "gn_silu on R256:" in msg, msg


def _no_rescale(q, k, v, H, D, scale, tile=128):
    """Online softmax over key tiles WITHOUT rescaling the running sums when the maximum grows:
    (o, lse) in fp64."""
    T, Tk = q.shape[1], k.shape[1]
    Q = q[0].to(ne.F64).reshape(T, H, D).transpose(0, 1)
    K = k[0].to(ne.F64).reshape(Tk, H, D).transpose(0, 1)
    V = v[0].to(ne.F64).reshape(Tk, H, D).transpose(0, 1)
    m = torch.full((H, T, 1), -math.inf, dtype=ne.F64)
    acc, l = torch.zeros(H, T, D, dtype=ne.F64), torch.zeros(H, T, 1, dtype=ne.F64)
    for j in range(0, Tk, tile):
        s = (Q @ K[:, j:j + tile].transpose(1, 2)) * scale
        m = torch.maximum(m, s.amax(-1, keepdim=True))
        p = torch.exp(s - m)                                   # alpha = exp(m_old - m_new) dropped
        l = l + p.sum(-1, keepdim=True)
        acc = acc + p @ V[:, j:j + tile]
    return (acc / l).transpose(0, 1).reshape(1, T, H * D), (m + torch.log(l))[..., 0][None]


def m_no_rescale(post, outs, pre):
    """attention's outputs written by the online softmax without its rescale."""
    o, lse = _no_rescale(pre["q"], pre["k"], pre["v"], pre["heads"], pre["head_dim"], pre["scale"])
    mid = pre["heads"] * pre["head_dim"]
    post["o"][..., :mid] = o.to(post["o"].dtype)
    if post["lse"] is not None:
        post["lse"].copy_(lse.to(post["lse"].dtype))


@pytest.mark.parametrize("D", [32, 64, 128])
def test_attention_check_passes_the_restatement(D):
    sh = ne.attention_case("late40", D, lambda: lc.Shadow(fake=True, probe=True), dev="cpu", backward=False)
    assert sh.n_checked == 1


@pytest.mark.parametrize("case", ["late40", "late80"])
def test_attention_without_rescale_fails(case):
    with pytest.raises(lc.CheckError, match="attention: o"):
        ne.attention_case(case, 64, lambda: lc.Shadow(fake=True, mutate=("attention", m_no_rescale)),
                          dev="cpu", backward=False)


def test_attention_without_rescale_is_exact_where_the_maximum_stays():
    """All-equal logits: the running maximum never moves, alpha = 1 is right, the check passes
    (the failures above are the rescale's, not the restatement's)."""
    sh = ne.attention_case("equal", 64, lambda: lc.Shadow(fake=True, mutate=("attention", m_no_rescale)),
                           dev="cpu", backward=False)
    assert sh.n_checked == 1
