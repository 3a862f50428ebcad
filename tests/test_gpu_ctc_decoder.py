"""cuda_ctc_decoder on the GPU.

* Against the float64 numpy oracle over the beam / V / threshold / skip / ragged-length / repeat matrix, on
  continuous random log-probabilities: tokens equal and scores within 1e-5 on every row whose decisions clear
  MARGIN, with at least one such row asserted per case.
* Against the numpy oracle (tests/ctc_decoder_oracle.py) on rows whose decision margins are all clear, including a
  prefix that leaves the beam, is re-created and must merge by string.
* Batch independence, offsets past 2^31 elements, errors and streams.
"""
import math

import numpy as np
import pytest
import torch

import ctc_decoder_oracle as O
from audio_b200.models.decoder import CUCTCDecoder, cuda_ctc_decoder

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def emissions(seed, B, T, V, skip=0.0, favour=0, scale=2.0):
    """log_softmax of N(0, scale) logits (float32).  A fraction `skip` of the frames get blank log-prob 0 (skipped
    at every threshold); `favour` > 0 boosts tokens 1..favour on every frame (heavy repeats, many merges)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, V, generator=g) * scale
    if favour:
        x[..., 1:favour + 1] += 4.0
    lp = torch.log_softmax(x, -1)
    if skip:
        lp[..., 0] = torch.where(torch.rand(B, T, generator=g) < skip, torch.zeros(()), lp[..., 0])
    return lp.numpy()


def spread_row(lp, b, seed):
    """Frame 0 of row b becomes distinct values 0.01 apart (blank at most -1, so selected at every threshold): a
    one-frame row whose top-`beam` decision clears any margin."""
    V = lp.shape[2]
    lp[b, 0] = -1.0 - 0.01 * np.random.default_rng(seed).permutation(V).astype(np.float32)


MARGIN = 2e-4  # well above the float32 rounding of a key, far below the gaps of these continuous inputs


def compare_with_oracle(lp, lens, beam, nbest, thr):
    """Each row of one batched call against the float64 oracle: on every row whose decisions all clear MARGIN, the
    same tokens at every position and scores within 1e-5 relative; rows with no selected frame empty with score 0.
    Returns the number of rows compared."""
    B, T, V = lp.shape
    vocab = [str(i) for i in range(V)]
    ours = cuda_ctc_decoder(vocab, nbest=nbest, beam_size=beam, blank_skip_threshold=thr)(
        torch.from_numpy(lp).to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV))
    log_thr = float(np.float32(math.log(thr)))
    compared = 0
    for b in range(B):
        assert len(ours[b]) == nbest
        for h in ours[b]:
            assert h.tokens.dtype == torch.int32 and h.score.dtype == torch.float32 and h.score.dim() == 0
            assert h.words == [vocab[t] for t in h.tokens.tolist()]
        hyps, margins = O.decode(lp[b].astype(np.float64), lens[b], beam, log_thr)
        if not hyps:
            assert all(h.tokens.numel() == 0 and h.score.item() == 0.0 for h in ours[b])
            continue
        if min(margins) <= MARGIN:
            continue
        compared += 1
        for h, (tok, score) in zip(ours[b], hyps):
            assert tuple(h.tokens.tolist()) == tok, (b, h.tokens.tolist(), tok)
            assert abs(h.score.item() - score) <= 1e-5 * max(1.0, abs(score)), (b, h.score.item(), score)
    return compared


@pytest.mark.parametrize("beam", [1, 2, 10, 64, 128])
@pytest.mark.parametrize("V", [2, 32, 500, 5000, 32000])
def test_beam_vocab_matrix(beam, V):
    if beam > V:
        pytest.skip("a beam above V raises ValueError (test_errors_and_empty_cases)")
    T = 40 if V >= 5000 else 96
    lp = emissions(1000 + beam * 7 + V, 5, T, V, skip=0.3)
    lens = [T, 0, T // 2, 1, T - 3]
    spread_row(lp, 3, V + beam)
    assert compare_with_oracle(lp, lens, beam, beam, 0.95) >= 1  # the one-frame row at least


@pytest.mark.parametrize("thr", [0.95, 0.5, 1.0])
@pytest.mark.parametrize("beam,V", [(10, 32), (64, 500), (4, 5)])
def test_thresholds_and_skips(thr, beam, V):
    T = 80
    lp = emissions(7 + beam + V, 4, T, V, skip=0.5)
    lp[1, :, 0] = 0.0   # every frame skipped
    lp[2, :, 0] = -3.0  # no frame skipped
    lp[3, :37, 0] = np.minimum(lp[3, :37, 0], -1.0)
    assert compare_with_oracle(lp, [T, T, T, 37], beam, min(beam, 3), thr) >= 1


@pytest.mark.parametrize("beam,V,favour", [(10, 32, 3), (16, 500, 4), (128, 500, 6), (2, 3, 2), (3, 3, 2)])
def test_repeats_and_merges(beam, V, favour):
    T = 120
    lp = emissions(55 + favour + beam, 4, T, V, skip=0.2, favour=favour)
    spread_row(lp, 3, V + beam)
    assert compare_with_oracle(lp, [T, T - 1, 60, 1], beam, beam, 0.95) >= 1


def test_recreated_prefix_merges_by_string():
    """Beam 3, V 3: "1 2" survives while "1" leaves the beam and is re-created from the empty prefix under a new trie
    node; "1" + 2 must then merge into "1 2" (the oracle counts such merges)."""
    r = np.random.default_rng(104)
    x = r.standard_normal((16, 3)) * 3
    x[:, 0] += (r.random(16) < 0.5) * 4
    lp = (x - np.logaddexp.reduce(x, axis=1, keepdims=True)).astype(np.float32)
    stats = {}
    hyps, margins = O.decode(lp.astype(np.float64), 16, 3, 0.0, stats=stats)
    assert stats["recreated_merges"] >= 1 and min(margins) > 0.1
    got = cuda_ctc_decoder(["-", "a", "b"], nbest=3, beam_size=3, blank_skip_threshold=1.0)(
        torch.from_numpy(lp[None]).to(DEV), torch.tensor([16], dtype=torch.int32, device=DEV))[0]
    for h, (tok, score) in zip(got, hyps):
        assert tuple(h.tokens.tolist()) == tok and abs(h.score.item() - score) <= 1e-5 * max(1.0, abs(score))


def peaky(seed, B, T, V):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, T, V, generator=g) * 2
    runs = torch.rand(B, T, generator=g) < 0.6
    logits[..., 0] += runs * 8.0
    tok = torch.randint(1, V, (B, T), generator=g)
    logits.scatter_add_(2, tok[..., None], (~runs)[..., None].float() * 6.0)
    return torch.log_softmax(logits, -1)


@pytest.mark.parametrize("seed,V,beam", [(11, 32, 10), (12, 500, 16), (13, 7, 4)])
def test_against_the_oracle(seed, V, beam):
    B, T = 4, 60
    lp = peaky(seed, B, T, V).numpy()
    lens = [T, 45, 1, 0]
    thr = 0.95
    ours = cuda_ctc_decoder([str(i) for i in range(V)], nbest=beam, beam_size=beam,
                            blank_skip_threshold=thr)(torch.from_numpy(lp).to(DEV), torch.tensor(lens, dtype=torch.int32, device=DEV))
    checked = 0
    for b in range(B):
        hyps, margins = O.decode(lp[b], lens[b], beam, float(np.float32(math.log(thr))))
        if not hyps:
            assert all(h.tokens.numel() == 0 and h.score.item() == 0.0 for h in ours[b])
            continue
        if min(margins) <= 1e-3:
            continue
        checked += 1
        for h, (tok, score) in zip(ours[b], hyps):
            assert tuple(h.tokens.tolist()) == tok
            assert abs(h.score.item() - score) <= 1e-4 * max(1.0, abs(score))
    assert checked >= 1


def test_batch_independence():
    V, T, beam = 500, 150, 10
    big = peaky(21, 128, T, V)
    lens = torch.randint(1, T + 1, (128,), generator=torch.Generator().manual_seed(3), dtype=torch.int32)
    dec = cuda_ctc_decoder([str(i) for i in range(V)], nbest=beam, beam_size=beam)
    x, n = big.to(DEV), lens.to(DEV)
    full = dec(x, n)
    for size in (1, 7, 128):
        part = dec(x[:size].contiguous(), n[:size].contiguous())
        for b in range(size):
            for h, g in zip(part[b], full[b]):
                assert torch.equal(h.tokens, g.tokens) and torch.equal(h.score, g.score)
    alone = dec(x[5:6].contiguous(), n[5:6].contiguous())
    for h, g in zip(alone[0], full[5]):
        assert torch.equal(h.tokens, g.tokens) and torch.equal(h.score, g.score)


def test_row_past_2_31_elements():
    V, T = 32768, 65537  # row 1 starts at 2^31 + 32768 elements
    B = 2
    x = torch.full((B, T, V), -30.0, device=DEV)
    x[:, :, 0] = 0.0  # every frame skipped ...
    small = peaky(31, 1, 40, 64)[0]
    x[1, 1000:1040, :64] = small.to(DEV)  # ... except 40 adjacent frames of row 1
    n = torch.tensor([T, T], dtype=torch.int32, device=DEV)
    dec = cuda_ctc_decoder([str(i) for i in range(V)], nbest=4, beam_size=4)
    got = dec(x, n)
    alone = dec(x[1:].contiguous(), n[1:].contiguous())
    hyps, margins = O.decode(x[1, 1000:1040].double().cpu().numpy(), 40, 4, float(np.float32(math.log(0.95))))
    del x
    torch.cuda.empty_cache()
    assert all(h.tokens.numel() == 0 and h.score.item() == 0.0 for h in got[0])
    for h, a in zip(got[1], alone[0]):
        assert torch.equal(h.tokens, a.tokens) and torch.equal(h.score, a.score)
    if min(margins) > 1e-3:
        for h, (tok, score) in zip(got[1], hyps):
            assert tuple(h.tokens.tolist()) == tok and abs(h.score.item() - score) <= 1e-4 * max(1.0, abs(score))


def test_errors_and_empty_cases():
    V, T = 8, 10
    x = torch.log_softmax(torch.randn(2, T, V, device=DEV), -1)
    dec = cuda_ctc_decoder([str(i) for i in range(V)], nbest=2, beam_size=4)
    with pytest.raises(ValueError, match="encoder_out_lens"):
        dec(x, torch.tensor([T + 1, 3], dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="encoder_out_lens"):
        dec(x, torch.tensor([2, -1], dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="beam_size"):
        cuda_ctc_decoder([str(i) for i in range(V + 4)], beam_size=12)(x, torch.tensor([T, T], dtype=torch.int32,
                                                                                         device=DEV))
    with pytest.raises(IndexError):
        cuda_ctc_decoder([str(i) for i in range(V)], nbest=5, beam_size=4)(x, torch.tensor([T, T], dtype=torch.int32,
                                                                                             device=DEV))
    assert dec(x[:0], torch.zeros(0, dtype=torch.int32, device=DEV)) == []
    empty = dec(torch.zeros(2, 0, V, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV))
    assert all(h.tokens.numel() == 0 and h.words == [] and h.score.item() == 0.0 for row in empty for h in row)
    with pytest.raises(RuntimeError, match="log_prob must be contiguous"):
        dec(x.transpose(0, 1), torch.tensor([T, T], dtype=torch.int32, device=DEV))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    on_stream = CUCTCDecoder([str(i) for i in range(V)], nbest=2, beam_size=4, cuda_stream=s)
    n = torch.tensor([T, 5], dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    a, b = dec(x, n), on_stream(x, n)
    for ra, rb in zip(a, b):
        for ha, hb in zip(ra, rb):
            assert torch.equal(ha.tokens, hb.tokens) and torch.equal(ha.score, hb.score)
