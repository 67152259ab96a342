"""adp_mel_spectrogram at STFT sizes other than powers of two (the mixed-radix FFT: every n_fft in
[32, 8192] with prime factors 2, 3, 5, 7) and with center=True:

  * the kernel against torchaudio's CPU route of the same module (rel-L2 1e-4, or in the log domain
    the pair used by test_frontend_gpu.py), at common vocoder sizes up to 8192 with hops that do not
    divide n_fft, shorter windows, normalize / normalize_log and frame counts not a multiple of 8;
  * center=True at a power of two and at other sizes against torchaudio, and its edge cases
    (a signal just long enough for both reflections, one frame) against an fp64 restatement;
  * refusals of n_fft outside the envelope on CUDA tensors, while CPU tensors keep torchaudio;
  * the non-power-of-two launches under the per-launch checker (tests/launch_check.py);
  * DiffusionVocoder at n_fft 400 and 1200 against the oracle port: loss, gradients, a 3-step sample.
Run with -s for the observed errors."""
import math

import pytest
import torch
import torch.nn.functional as F

import launch_check as lc

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRAD_TOL = 6e-2                     # DESIGN.md section 2: bf16 storage, parameter gradients


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def close(got, want, log):
    """rel-L2 1e-4; log(max(mel, 1e-5)) is compared where the clamp is inactive (exp) and absolutely."""
    if log:
        e_abs, e = float((got.cpu() - want).abs().max()), rel_l2(got.exp(), want.exp())
        assert e_abs <= 2e-3 and e <= 1e-4, (e_abs, e)
        return f"rel-L2(exp) {e:.2e}, max |log err| {e_abs:.2e}"
    e = rel_l2(got, want)
    assert e <= 1e-4, e
    return f"rel-L2 {e:.2e}"


# n_fft, hop, win_length, n_mels, sample_rate, extra module options
SIZES = {
    400: (400, 160, 400, 80, 16000, {}),                          # hop does not divide n_fft
    441: (441, 110, 441, 64, 44100, {}),                          # odd: 221 bins
    480: (480, 120, 400, 80, 48000, {}),                          # win_length < n_fft
    800: (800, 200, 800, 80, 16000, dict(normalize=True)),
    882: (882, 300, 882, 80, 44100, dict(normalize_log=True)),
    1200: (1200, 300, 1200, 128, 48000, {}),
    1323: (1323, 331, 1000, 80, 44100, dict(normalize_log=True)),  # odd, odd window offset
    1920: (1920, 480, 1920, 128, 48000, dict(normalize=True, normalize_log=True)),
    2000: (2000, 500, 1600, 80, 16000, {}),
    3000: (3000, 700, 3000, 160, 48000, dict(normalize_log=True)),
    6000: (6000, 1500, 6000, 256, 48000, {}),
    8192: (8192, 2048, 8192, 512, 48000, dict(normalize_log=True)),  # the largest FFT, 512 mels
}


@pytest.mark.parametrize("n_fft", list(SIZES))
def test_mel_spectrogram_sizes(n_fft):
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    n_fft, hop, win, n_mels, sr, extra = SIZES[n_fft]
    torch.manual_seed(1)
    front = MelSpectrogram(n_fft=n_fft, hop_length=hop, win_length=win, sample_rate=sr, n_mel_channels=n_mels,
                           **extra)
    t = 2 ** 15
    wave = torch.randn(2, 2, t) * torch.linspace(0.05, 1.0, t)
    log = extra.get("normalize_log", False) and not extra.get("normalize", False)
    want = front(wave)
    got = front.to(DEV)(wave.to(DEV))
    assert got.shape == want.shape
    msg = close(got, want, log)
    odd = wave[..., : t - 123 * 7]
    frames = 1 + (odd.shape[-1] + 2 * front.padding - n_fft) // hop
    got_odd = front(odd.to(DEV))
    assert got_odd.shape[-1] == frames
    if frames % 8 == 0:                 # keep the partial last CTA covered
        odd = odd[..., :-hop]
        got_odd = front(odd.to(DEV))
    assert got_odd.shape[-1] % 8 != 0
    msg_odd = close(got_odd, front.cpu()(odd), log)
    print(f"\nn_fft {n_fft}: {msg}; {got_odd.shape[-1]} frames: {msg_odd}")


@pytest.mark.parametrize("n_fft,hop,win,log", [(1024, 256, 1024, False), (512, 128, 400, True),
                                               (441, 110, 441, False), (1200, 300, 1200, True),
                                               (1920, 480, 1500, False)])
def test_center_true_against_torchaudio(n_fft, hop, win, log):
    """MelSpectrogram(center=True): the module's reflect pad by (n_fft - hop) // 2, then torch.stft's
    own reflect pad by n_fft // 2; the kernel gets the second as center_pad."""
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    torch.manual_seed(2)
    front = MelSpectrogram(n_fft=n_fft, hop_length=hop, win_length=win, sample_rate=48000, n_mel_channels=64,
                           center=True, normalize_log=log)
    wave = torch.randn(3, 5000) * torch.linspace(1.0, 0.1, 5000)
    want = front(wave)
    got = front.to(DEV)(wave.to(DEV))
    assert got.shape == want.shape
    assert got.shape[-1] == 1 + (5000 + 2 * front.padding + 2 * (n_fft // 2) - n_fft) // hop
    print(f"\ncenter=True n_fft {n_fft}: {close(got, want, log)}")


def fp64_mel(wave, window, fb, n_fft, hop, pad, center_pad):
    """Reflect-pad by pad, reflect-pad that by center_pad, frames, window, rfft, |.|, fb, in fp64."""
    x = F.pad(wave.double()[:, None], (pad, pad), mode="reflect")
    x = F.pad(x, (center_pad, center_pad), mode="reflect")[:, 0]
    fr = x.unfold(-1, n_fft, hop) * window.double()
    return (torch.fft.rfft(fr, dim=-1).abs() @ fb.double()).transpose(1, 2)


# n_fft, hop, win_length, t: the shortest signals both reflections accept, and a single frame
CENTER_EDGES = {
    "just_long_enough_400": (400, 100, 400, 151),        # pad 150 < t = 151; center_pad 200 < t + 300
    "just_long_enough_1024": (1024, 256, 800, 385),      # pad 384, center_pad 512
    "one_frame_441": (441, 441, 441, 221),               # pad 0, center_pad 220 < t = 221: frames 1
    "one_frame_2000": (2000, 2000, 1600, 1001),          # pad 0, center_pad 1000
}


@pytest.mark.parametrize("name", list(CENTER_EDGES))
def test_center_edges_against_fp64(name):
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    n_fft, hop, win, t = CENTER_EDGES[name]
    front = MelSpectrogram(n_fft=n_fft, hop_length=hop, win_length=win, sample_rate=16000, n_mel_channels=40,
                           center=True)
    window, fb, band = front._kernel_tables(DEV)
    pad, cpad = front.padding, n_fft // 2
    assert pad < t and cpad < t + 2 * pad
    wave = torch.randn(3, t, generator=torch.Generator().manual_seed(3)) * torch.arange(1, 4)[:, None]
    got = ops.mel_spectrogram(wave.to(DEV), window, fb, band, n_fft, hop, pad, apply_log=False, center_pad=cpad)
    want = fp64_mel(wave, window.cpu(), fb.cpu(), n_fft, hop, pad, cpad)
    assert got.shape == want.shape
    if name.startswith("one_frame"):
        assert got.shape[-1] == 1
    e = rel_l2(got, want)
    # the same through the module (CUDA route) and torchaudio's CPU route
    e_mod = rel_l2(front(wave.to(DEV)), front.cpu()(wave))
    print(f"\n{name}: rel-L2 {e:.2e} vs fp64, module vs torchaudio {e_mod:.2e}")
    assert e <= 1e-5 and e_mod <= 1e-4


@pytest.mark.parametrize("n_fft", [1102, 2002, 16384])
def test_sizes_outside_the_envelope_are_refused_on_cuda(n_fft):
    """1102 = 2 * 19 * 29, 2002 = 2 * 7 * 11 * 13 and 16384 raise on CUDA tensors with the limit named;
    the same module on CPU tensors returns torchaudio's result."""
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    front = MelSpectrogram(n_fft=n_fft, hop_length=n_fft // 4, win_length=n_fft, sample_rate=48000,
                           n_mel_channels=64)
    wave = torch.randn(2, 3 * n_fft, generator=torch.Generator().manual_seed(4))
    want = front(wave)
    flat = F.pad(wave, [front.padding] * 2, mode="reflect")
    assert torch.equal(want, front.to_mel_scale(torch.abs(front.to_spectrogram(flat))))
    with pytest.raises(RuntimeError, match=rf"n_fft={n_fft} must have prime factors 2, 3, 5, 7 only and lie in "
                                           r"\[32, 8192\]"):
        front.to(DEV)(wave.to(DEV))
    assert torch.equal(front.cpu()(wave), want)


def test_pads_longer_than_the_signal_are_refused():
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    front = MelSpectrogram(n_fft=400, hop_length=100, win_length=400, sample_rate=16000, n_mel_channels=40)
    window, fb, band = front._kernel_tables(DEV)
    wave = torch.randn(1, 150, device=DEV)                 # pad 150 is not shorter than t
    with pytest.raises(RuntimeError, match="shorter than the signal it mirrors"):
        ops.mel_spectrogram(wave, window, fb, band, 400, 100, 150, apply_log=False)
    wave = torch.randn(1, 60, device=DEV)                  # center_pad 200 >= t + 2 pad = 180
    with pytest.raises(RuntimeError, match="shorter than the signal it mirrors"):
        ops.mel_spectrogram(wave, window, fb, band, 400, 100, 60 - 1, apply_log=False, center_pad=200)


# (n_fft, hop, win_length, n_mels, sample_rate, t, log)
CHECKED = {
    "n_fft400": (400, 100, 400, 80, 16000, 8000, True),
    "n_fft441_odd": (441, 110, 441, 64, 44100, 5003, False),
    "n_fft1323_win1000": (1323, 331, 1000, 80, 44100, 20000, True),
    "n_fft1920": (1920, 480, 1920, 128, 48000, 2 ** 15, True),
    "n_fft3000_hop700": (3000, 700, 3000, 160, 48000, 30011, False),
    "n_fft6561_radix3": (6561, 1640, 6561, 128, 48000, 2 ** 15, True),
    "n_fft8192_mels512": (8192, 2048, 8192, 512, 48000, 2 ** 16, True),
    "n_fft2205_frames1": (2205, 512, 2205, 64, 44100, 900, False),          # pad 846 < t = 900
}


def test_non_power_of_two_launches_checked():
    """Direct launches (center_pad 0) under lc.Shadow: every output element against the fp64
    restatement c_mel_spectrogram, with its per-element bound."""
    from audio_diffusion_pytorch_b200 import ops
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    ops.device_check()
    g = torch.Generator().manual_seed(8)
    with lc.Shadow() as sh:
        for name, (n_fft, hop, win, n_mels, sr, t, log) in CHECKED.items():
            front = MelSpectrogram(n_fft=n_fft, hop_length=hop, win_length=win, sample_rate=sr, n_mel_channels=n_mels)
            window, fb, band = front._kernel_tables(DEV)
            wave = (torch.randn(3, t, generator=g) * torch.arange(1, 4)[:, None]).to(DEV)
            mel = ops.mel_spectrogram(wave, window, fb, band, n_fft, hop, front.padding, apply_log=log)
            if name.endswith("frames1"):
                assert mel.shape[-1] == 1
    print(f"\n{sh.table()}")
    assert sh.n_checked == sh.n_launch == len(CHECKED)


def _compare_grads(ref_params, got_params):
    """Worst per-parameter rel-L2 (floored as in test_train_gpu.py) and the global cosine."""
    norms = torch.stack([p.grad.double().norm() for _, p in ref_params])
    floor = max(0.1 * float(norms.median()), 1e-3 * float(norms.max()))
    worst, dots, n1, n2 = 0.0, 0.0, 0.0, 0.0
    for (name, p), q in zip(ref_params, got_params):
        assert q.grad is not None, f"no gradient for {name}"
        g_ref, g = p.grad.double(), q.grad.double().cpu()
        worst = max(worst, float((g - g_ref).norm() / g_ref.norm().clamp_min(floor)))
        dots += float((g * g_ref).sum())
        n1 += float((g * g).sum())
        n2 += float((g_ref * g_ref).sum())
    return worst, dots / math.sqrt(n1 * n2)


@pytest.mark.parametrize("n_fft,hop,t", [(400, 100, 8000), (1200, 300, 12000)])
def test_vocoder_against_oracle(oracle_port, n_fft, hop, t):
    """DiffusionVocoder at a non-power-of-two n_fft: the training loss (mel kernel, to_flat, fused
    loss and backward), every parameter gradient and to_flat.weight.grad, and a 3-step sample,
    against the oracle port with the same weights and draws."""
    import audio_diffusion_pytorch_b200 as adp
    kw = dict(mel_n_fft=n_fft, mel_hop_length=hop, mel_channels=80, mel_sample_rate=48000, mel_normalize_log=True,
              channels=[8, 32], factors=[1, 4], items=[1, 1])
    torch.manual_seed(0)
    ref = oracle_port.DiffusionVocoderPort(**kw)
    model = adp.DiffusionVocoder(net_t=adp.UNetV0, **kw).to(DEV)
    model.net.load_reference_parameters(ref.net)
    model.to_flat.load_state_dict(ref.to_flat.state_dict())
    audio = torch.randn(2, 2, t, generator=torch.Generator().manual_seed(9))
    torch.manual_seed(31)
    loss = model(audio.to(DEV))
    loss.backward()
    torch.manual_seed(31)                       # the same sigma / noise draws (GPU generator, rows = b*c)
    sigma = torch.rand(4, device=DEV).cpu()
    noise = torch.randn(4, 1, t, device=DEV).cpu()
    mel = ref.to_spectrogram(audio)
    guide = ref.to_flat(mel.reshape(-1, *mel.shape[-2:]))
    assert guide.shape[-1] == t
    rows = audio.reshape(-1, 1, t)
    a, b = torch.cos(sigma * math.pi / 2)[:, None, None], torch.sin(sigma * math.pi / 2)[:, None, None]
    loss_ref = F.mse_loss(ref.net(a * rows + b * noise, sigma, append_channels=guide), a * noise - b * rows)
    loss_ref.backward()
    rel = abs(float(loss.detach()) - float(loss_ref.detach())) / float(loss_ref.detach())
    e_flat = rel_l2(model.to_flat.weight.grad, ref.to_flat.weight.grad)
    gw, gf = model.to_flat.weight.grad.double().flatten().cpu(), ref.to_flat.weight.grad.double().flatten()
    cos_flat = float(gw @ gf / (gw.norm() * gf.norm()))
    worst, cos = _compare_grads(list(ref.net.named_parameters()), list(model.net.parameters()))
    with torch.no_grad():
        s = model.sample(mel.to(DEV), num_steps=3, generator=torch.Generator().manual_seed(8))
        s_ref = ref.sample(mel, num_steps=3, generator=torch.Generator().manual_seed(8))
    e_s = rel_l2(s, s_ref)
    print(f"\nvocoder n_fft {n_fft}: loss rel {rel:.2e}; to_flat.weight.grad rel-L2 {e_flat:.2e} "
          f"(cos {cos_flat:.6f}); worst parameter gradient {worst:.2e} (global cos {cos:.6f}); "
          f"3-step sample {e_s:.2e}")
    assert rel < 2e-3
    assert e_flat < GRAD_TOL and cos_flat >= 0.999
    assert worst < GRAD_TOL and cos >= 0.999
    assert s.shape == s_ref.shape and e_s <= 5e-3
