"""Host side of adp_mel_spectrogram at STFT sizes other than powers of two (odd n_fft has
n_fft // 2 + 1 bins, a shorter window is centred the way torch.stft centres it), and the CPU
route of MelSpectrogram / DiffusionVocoder at those sizes, which stays torchaudio's."""
import pytest
import torch
import torch.nn.functional as F

# (n_fft, win_length, n_mels, sample_rate)
SIZES = [(400, 400, 80, 16000), (441, 441, 64, 44100), (441, 300, 64, 44100), (1323, 1024, 80, 44100),
         (2205, 2000, 128, 44100), (1200, 1199, 128, 48000), (6000, 4800, 256, 48000), (8192, 8192, 512, 48000)]


@pytest.mark.parametrize("n_fft,win,n_mels,sr", SIZES)
def test_kernel_tables_at_any_n_fft(n_fft, win, n_mels, sr):
    """The window handed to the kernel is the module's window padded to n_fft exactly where
    torch.stft puts it (so framing with it equals torch.stft with the short window), and every
    mel filter's non-zero bins lie inside its [lo, hi) range, so the banded product equals the
    full filterbank matmul."""
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    front = MelSpectrogram(n_fft=n_fft, hop_length=n_fft // 4 + 1, win_length=win, sample_rate=sr,
                           n_mel_channels=n_mels)
    window, fb, band = front._kernel_tables(torch.device("cpu"))
    bins = n_fft // 2 + 1
    assert window.shape == (n_fft,) and fb.shape == (bins, n_mels) and band.shape == (n_mels, 2)
    left = (n_fft - win) // 2
    assert torch.equal(window[left:left + win], front.to_spectrogram.window)
    assert float(window[:left].abs().sum() + window[left + win:].abs().sum()) == 0.0
    x = torch.randn(3 * n_fft, dtype=torch.float64)
    want = torch.stft(x, n_fft, hop_length=n_fft // 3, win_length=win, window=front.to_spectrogram.window.double(),
                      center=False, return_complex=True)
    got = torch.stft(x, n_fft, hop_length=n_fft // 3, window=window.double(), center=False, return_complex=True)
    assert want.shape[0] == bins
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    mag = torch.rand(bins)
    full = mag @ fb
    banded = torch.stack([(mag[lo:hi] * fb[lo:hi, m]).sum() for m, (lo, hi) in enumerate(band.tolist())])
    assert torch.allclose(banded, full, rtol=1e-6, atol=1e-7)
    for m, (lo, hi) in enumerate(band.tolist()):
        assert 0 <= lo <= hi <= bins
        nz = torch.nonzero(fb[:, m]).flatten()
        if nz.numel() == 0:
            assert lo == hi
        else:
            assert lo <= int(nz.min()) and int(nz.max()) < hi


@pytest.mark.parametrize("n_fft,hop,center", [(400, 100, False), (441, 110, True), (1102, 256, False),
                                              (16384, 4096, True)])
def test_cpu_route_is_torchaudio_at_any_n_fft(oracle_port, n_fft, hop, center):
    """Host tensors keep the tensor-op route at any n_fft, including sizes the kernel refuses
    (1102 = 2 * 19 * 29, 16384): the module's output is the reference module's."""
    from audio_diffusion_pytorch_b200.components import MelSpectrogram
    kw = dict(n_fft=n_fft, hop_length=hop, win_length=n_fft, sample_rate=44100, n_mel_channels=40,
              center=center, normalize_log=True)
    wave = torch.randn(2, 2, 3 * n_fft, generator=torch.Generator().manual_seed(0))
    got = MelSpectrogram(**kw)(wave)
    want = oracle_port.MelSpectrogramPort(**kw)(wave)
    assert torch.equal(got, want)
    frames = 1 + (3 * n_fft + 2 * ((n_fft - hop) // 2) + 2 * (n_fft // 2 if center else 0) - n_fft) // hop
    assert got.shape == (2, 2, 40, frames)


def test_vocoder_on_cpu_at_a_non_power_of_two_n_fft(oracle_port):
    """A DiffusionVocoder whose net is not the CUDA U-Net trains on the CPU at n_fft 400: the
    front-end and to_flat take the tensor-op route and equal the reference's, and the training step
    gives to_flat a gradient."""
    import audio_diffusion_pytorch_b200 as adp
    kw = dict(mel_n_fft=400, mel_hop_length=100, mel_channels=16, mel_sample_rate=16000,
              channels=[8, 32], factors=[1, 4], items=[1, 1])
    torch.manual_seed(0)
    ref = oracle_port.DiffusionVocoderPort(**kw)
    voc = adp.DiffusionVocoder(net_t=oracle_port.build_unet_v0, **kw)
    voc.to_flat.load_state_dict(ref.to_flat.state_dict())
    audio = torch.randn(2, 1, 8000, generator=torch.Generator().manual_seed(1))
    mel = voc.to_spectrogram(audio)
    assert mel.shape == (2, 1, 16, 80)
    assert torch.equal(mel, ref.to_spectrogram(audio))
    guide, lead = voc._unroll(mel)
    assert lead == (2, 1) and torch.equal(guide, ref.to_flat(mel.reshape(-1, 16, 80)))
    loss = voc(audio)
    loss.backward()
    assert torch.isfinite(loss) and voc.to_flat.weight.grad is not None


def test_double_reflection_is_not_one_reflection():
    """center=True after the module's pad reflects twice (F.pad, then torch.stft's own pad).  Near the
    ends that reads other samples than one reflection by the summed pad, which is why the kernel
    composes the two index maps: pinned here on the index arithmetic the kernel uses."""
    def reflect(j, n):
        return torch.where(j < 0, -j, torch.where(j >= n, 2 * (n - 1) - j, j))

    t, pad, cpad = 37, 9, 20
    x = torch.arange(t, dtype=torch.float64)
    twice = F.pad(F.pad(x[None, None], (pad, pad), mode="reflect"), (cpad, cpad), mode="reflect")[0, 0]
    j = torch.arange(t + 2 * pad + 2 * cpad)
    composed = x[reflect(reflect(j - cpad, t + 2 * pad) - pad, t)]
    assert torch.equal(composed, twice)
    once = F.pad(x[None, None], (pad + cpad, pad + cpad), mode="reflect")[0, 0]
    assert not torch.equal(once, twice)
