"""The device PNG decoder (csrc/png_decode.cu) against cv2.imread on the corpus of tests/golden/reference_png_v1.npz: bit for bit, in
one launch and in shuffled sub-batches; the malformed set gives the host decoder's statuses; encode_png -> decode_png round trips."""
import os

import numpy as np
import pytest
import torch

from ssdnerf_b200 import datasets as D

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_png_v1.npz')


@pytest.fixture(scope='module')
def png():
    return np.load(GOLDEN)


def corpus(npz, prefix):
    b, o = npz[f'{prefix}_bytes'], npz[f'{prefix}_offsets']
    return [(str(n), b[o[i]:o[i + 1]].tobytes()) for i, n in enumerate(npz[f'{prefix}_names'])]


def expected(npz):
    shapes = npz['valid_shapes']
    po = np.cumsum([0] + [int(np.prod(s)) for s in shapes])
    return [npz['valid_pixels'][po[i]:po[i + 1]].reshape(shapes[i]).astype(np.float32) / 255 for i in range(len(shapes))]


def test_corpus_in_one_call_and_in_shuffled_sub_batches(cuda, png):
    files, want = corpus(png, 'valid'), expected(png)
    names = [n for n, _ in files]
    got = D.decode_png_images([f for _, f in files], cuda, names)
    for n, g, w in zip(names, got, want):
        assert np.array_equal(g.cpu().numpy(), w), n
    rng = np.random.default_rng(5)
    order = rng.permutation(len(files))
    for part in np.array_split(order, 7):
        sub = D.decode_png_images([files[i][1] for i in part], cuda, [names[i] for i in part])
        for i, g in zip(part, sub):
            assert torch.equal(g, got[i]), names[i]


def test_stacked_batch_of_one_size(cuda, png):
    files, want = corpus(png, 'valid'), expected(png)
    idx = [i for i, w in enumerate(want) if w.shape == (128, 128, 3)]
    assert len(idx) >= 30
    out = D.decode_png([files[i][1] for i in idx], cuda, [files[i][0] for i in idx])
    assert out.shape == (len(idx), 128, 128, 3) and out.dtype == torch.float32
    assert np.array_equal(out.cpu().numpy(), np.stack([want[i] for i in idx]))


def test_malformed_set_statuses_match_the_host_decoder(cuda, png):
    mal = [(n, f, s) for (n, f), s in zip(corpus(png, 'mal'), png['mal_status']) if s >= 0]
    good = corpus(png, 'valid')[:3]
    batch = good + [(n, f) for n, f, _ in mal]
    infos = [D.parse_png(f, n) for n, f in batch]
    _, _, st = D._decode(infos, cuda)
    host = [D.decode_png_host(f, n)[1] for n, f in batch]
    assert st.tolist() == host
    assert st.tolist() == [0, 0, 0] + [int(s) for _, _, s in mal]
    with pytest.raises(ValueError, match=f'{mal[0][0]}: corrupt PNG data'):
        D.decode_png_images([f for _, f in batch], cuda, [n for n, _ in batch])


def test_encode_png_round_trip(cuda):
    from ssdnerf_b200 import viz
    g = torch.Generator().manual_seed(11)
    u8 = torch.randint(0, 256, (6, 40, 52, 3), generator=g, dtype=torch.uint8)
    u8[:, 10:30] = 200                                  # runs for the encoder's matches
    x = (u8.float() / 255).to(cuda)
    files = viz.encode_png(pred=x)
    out = D.decode_png(files, cuda)
    assert torch.equal(out, x)
