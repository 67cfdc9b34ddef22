"""Batched label-map consumers on the GPU (BaseSlic.get_connectivity_batch / get_mask_density_batch /
broadcast_density_to_mask_batch): every image of a batch equals the reference's fast_slic_get_connectivity,
fast_slic_get_mask_density and fast_slic_cluster_density_to_mask for that image alone, at tolerance 0 -- neighbour
order, the 12-neighbour cap and the table-overflow replay included."""
import numpy as np
import pytest
import torch

from cases import make_image

pytestmark = pytest.mark.gpu


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _struct(cl):
    from fast_slic_b200 import CLUSTER_DTYPE
    cl = _np(cl)
    return cl if cl.dtype == CLUSTER_DTYPE else np.ascontiguousarray(cl).view(CLUSTER_DTYPE).reshape(cl.shape[:2])


def _run(s, labels, masks, clusters):
    counts, nb, rep = s.get_connectivity_batch(labels, return_replayed=True)
    dens = s.get_mask_density_batch(masks, labels, clusters)
    bc = s.broadcast_density_to_mask_batch(dens, labels)
    return counts, nb, rep, dens, bc


def _host(outs):
    if isinstance(outs[0], torch.Tensor):
        torch.cuda.synchronize()
    return [_np(x) for x in outs]


def _check(checker, K, labels, masks, clusters, outs, replayed=None):
    """Image by image against the checker; `replayed`: the expected overflow flags (default: none)."""
    labels, masks, cl = _np(labels), _np(masks), _struct(clusters)
    counts, nb, rep, dens, bc = _host(outs)
    B = labels.shape[0]
    assert counts.shape == (B, K) and nb.shape == (B, K, 12) and dens.shape == (B, K) and bc.shape == labels.shape
    assert counts.dtype == np.int32 and nb.dtype == np.int32 and dens.dtype == np.uint8 and bc.dtype == np.uint8
    assert rep.tolist() == (replayed if replayed is not None else [0] * B)
    from fast_slic_b200 import NodeConnectivity
    for b in range(B):
        lab = labels[b].view(np.uint16)
        assert NodeConnectivity(counts[b], nb[b]).tolist() == checker.get_connectivity(lab, K), b
        assert (nb[b][np.arange(12)[None, :] >= counts[b][:, None]] == 0).all(), b
        assert (dens[b] == checker.get_mask_density(cl[b], lab, masks[b])).all(), b
        assert (bc[b] == checker.density_to_mask(K, lab, dens[b])).all(), b


def _slic_batch(H, W, K, B, msf, seed=0, kind="syn"):
    from fast_slic_b200 import Slic
    s = Slic(num_components=K, min_size_factor=msf)
    imgs = torch.from_numpy(np.stack([make_image(kind, H, W, seed=seed + b) for b in range(B)])).cuda()
    labels, clusters = s.iterate_batch(imgs, return_clusters=True)
    masks = torch.from_numpy(np.random.RandomState(seed + 99).randint(0, 256, (B, H, W)).astype(np.uint8)).cuda()
    return s, labels, masks, clusters


@pytest.fixture(scope="module", params=[0.0, 0.25], ids=["msf0", "msf.25"])
def superpixels(request):
    return _slic_batch(240, 320, 300, 8, request.param, seed=11)


def test_per_image_equals_the_reference(checker, superpixels):
    from fast_slic_b200 import SlicModel
    s, labels, masks, clusters = superpixels
    outs = _run(s, labels, masks, clusters)
    assert all(isinstance(x, torch.Tensor) and x.device == labels.device for x in outs)
    _check(checker, 300, labels, masks, clusters, outs)
    # ... and each image equals the single-image SlicModel methods
    counts, nb, _, dens, bc = _host(outs)
    lab, msk, cl = _np(labels), _np(masks), _struct(clusters)
    for b in range(lab.shape[0]):
        m = SlicModel(300)
        m._clusters = cl[b].copy()
        assert m.get_connectivity(lab[b]).tolist() == [nb[b, k, :counts[b, k]].tolist() for k in range(300)]
        assert (m.get_mask_density(msk[b], lab[b]) == dens[b]).all()
        assert (m.broadcast_density_to_mask(dens[b], lab[b]) == bc[b]).all()


def test_overflowing_image_replays_alone(checker):
    """K = 300 on 512x512 noise: far more distinct adjacent pairs than the 16384-slot table holds."""
    s, labels, masks, clusters = _slic_batch(512, 512, 300, 3, 0.0, seed=5)
    noise = torch.from_numpy(np.random.RandomState(4).randint(0, 300, (1, 512, 512)).astype(np.int16)).cuda()
    labels = torch.cat([labels[:1], noise, labels[1:]])
    masks = torch.cat([masks[:1], masks[:1].flip(1), masks[1:]])
    clusters = torch.cat([clusters[:1], clusters[2:3], clusters[1:]])
    _check(checker, 300, labels, masks, clusters, _run(s, labels, masks, clusters), replayed=[0, 1, 0, 0])


def test_labels_outside_the_range_are_ignored(checker):
    s, labels, masks, clusters = _slic_batch(97, 131, 60, 3, 0.0, seed=7)
    lab = _np(labels).copy()
    lab[0, ::7, ::5] = -1
    lab[1, 3::4, ::3] = 60
    lab[1, ::9, 2::6] = 30000
    lab[2, :, :] = -1
    lab = torch.from_numpy(lab).cuda()
    _check(checker, 60, lab, masks, clusters, _run(s, lab, masks, clusters))


@pytest.mark.parametrize("H,W", [(1, 50), (50, 1), (1, 1)])
def test_single_row_or_column_gives_empty_lists(checker, H, W):
    from fast_slic_b200 import Slic
    K, B = 20, 3
    rng = np.random.RandomState(H * 100 + W)
    s = Slic(num_components=K)
    lab = torch.from_numpy(rng.randint(-1, K, (B, H, W)).astype(np.int16)).cuda()
    masks = torch.from_numpy(rng.randint(0, 256, (B, H, W)).astype(np.uint8)).cuda()
    cl = _random_clusters(rng, B, K)
    outs = _run(s, lab, masks, cl)
    assert (_np(outs[0]) == 0).all()
    _check(checker, K, lab, masks, cl, outs)


def _random_clusters(rng, B, K, zero_every=0, members=None):
    from fast_slic_b200 import CLUSTER_DTYPE
    cl = np.zeros((B, K), CLUSTER_DTYPE)
    cl["num_members"] = rng.randint(0, 40, (B, K)) if members is None else members[None]
    if zero_every:
        cl["num_members"][:, ::zero_every] = 0
    cl["number"] = np.arange(K)[None]
    return torch.from_numpy(cl.view(np.uint8).reshape(B, K, 32).copy()).cuda()


@pytest.mark.parametrize("K,H,W,B", [(1, 40, 37, 3), (65533, 256, 256, 2)])
def test_smallest_and_largest_component_counts(checker, K, H, W, B):
    from fast_slic_b200 import Slic
    rng = np.random.RandomState(K)
    s = Slic(num_components=K)
    lo = -1 if K == 1 else 0
    lab = torch.from_numpy(rng.randint(lo, K, (B, H, W)).astype(np.uint16).view(np.int16)).cuda()
    masks = torch.from_numpy(rng.randint(0, 256, (B, H, W)).astype(np.uint8)).cuda()
    cl = _random_clusters(rng, B, K, zero_every=3)
    _check(checker, K, lab, masks, cl, _run(s, lab, masks, cl))


def test_twelve_neighbour_cap_and_empty_clusters(checker):
    """Few labels scattered at random: nearly every label meets more than 12 others, so the cap decides the lists;
    every third cluster record has num_members 0 (the density divides by 1 there)."""
    from fast_slic_b200 import Slic
    K, B, H, W = 48, 4, 120, 160
    rng = np.random.RandomState(3)
    s = Slic(num_components=K)
    lab = torch.from_numpy(rng.randint(0, 40, (B, H, W)).astype(np.int16)).cuda()
    masks = torch.from_numpy(rng.randint(0, 256, (B, H, W)).astype(np.uint8)).cuda()
    cl = _random_clusters(rng, B, K, zero_every=3)
    outs = _run(s, lab, masks, cl)
    assert (_np(outs[0]) == 12).sum() >= 4 * B
    _check(checker, K, lab, masks, cl, outs)


@pytest.mark.parametrize("H,W,B", [(97, 131, 5), (3, 5, 7), (1, 7, 9)])
def test_warps_straddling_images(checker, H, W, B):
    """H*W not a multiple of 32: a warp holds pixels of two or more images.  Every image has the same label map and
    its own mask, so sums merged across images would show.  num_members holds the true pixel counts, so the densities
    are the masks' means per label and do not saturate."""
    from fast_slic_b200 import Slic
    K = 6
    rng = np.random.RandomState(H + W)
    s = Slic(num_components=K)
    one = rng.randint(0, K, (H, W))
    lab = torch.from_numpy(np.repeat(one[None], B, 0).astype(np.int16)).cuda()
    masks = torch.from_numpy(rng.randint(0, 256, (B, H, W)).astype(np.uint8)).cuda()
    cl = _random_clusters(rng, B, K, members=np.bincount(one.ravel(), minlength=K))
    outs = _run(s, lab, masks, cl)
    assert len({_np(outs[3])[b].tobytes() for b in range(B)}) > 1
    _check(checker, K, lab, masks, cl, outs)


def test_empty_and_single_image_batches(checker, superpixels):
    s, labels, masks, clusters = superpixels
    counts, nb, rep, dens, bc = _run(s, labels[:0], masks[:0], clusters[:0])
    assert counts.shape == (0, 300) and nb.shape == (0, 300, 12) and rep.shape == (0,) and dens.shape == (0, 300)
    assert bc.shape == (0, 240, 320)
    counts, nb, rep, dens, bc = _host(_run(s, labels[:0].cpu().numpy(), masks[:0].cpu().numpy(), _struct(clusters)[:0]))
    assert counts.shape == (0, 300) and bc.shape == (0, 240, 320)
    _check(checker, 300, labels[2:3], masks[2:3], clusters[2:3], _run(s, labels[2:3], masks[2:3], clusters[2:3]))


def test_large_images(checker):
    s, labels, masks, clusters = _slic_batch(2160, 3840, 4000, 4, 0.25, seed=21, kind="tiled")
    _check(checker, 4000, labels, masks, clusters, _run(s, labels, masks, clusters))


def test_images_are_independent(superpixels, monkeypatch):
    from fast_slic_b200 import _lib, graph_batch
    s, labels, masks, clusters = superpixels
    want = _host(_run(s, labels, masks, clusters))
    perm = torch.tensor([5, 2, 7, 0, 3, 6, 1, 4], device=labels.device)
    got = _host(_run(s, labels[perm], masks[perm], clusters[perm]))
    p = perm.cpu().numpy()
    for w, g in zip(want, got):
        assert (w[p] == g).all()
    # a small scratch cap: the graph runs in chunks of at most three images
    monkeypatch.setattr(graph_batch, "GRAPH_SCRATCH_CAP", 3 * _lib.lib().fslic_b200_connectivity_batch_scratch_bytes(300, 1))
    assert graph_batch.graph_chunk(300, 8) <= 3
    got = _host(_run(s, labels, masks, clusters))
    for w, g in zip(want, got):
        assert (w == g).all()


def test_cuda_graph_capture_and_replay(superpixels):
    """No host synchronisation: the three calls capture into a CUDA graph; a replay on new inputs equals eager calls."""
    s, labels, masks, clusters = superpixels
    st_lab, st_mask, st_cl = labels.clone(), masks.clone(), clusters.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _run(s, st_lab, st_mask, st_cl)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static_out = _run(s, st_lab, st_mask, st_cl)
    # new inputs: another batch's superpixels
    _, labels2, masks2, clusters2 = _slic_batch(240, 320, 300, 8, 0.0, seed=40)
    st_lab.copy_(labels2)
    st_mask.copy_(masks2)
    st_cl.copy_(clusters2)
    g.replay()
    got = _host(static_out)
    want = _host(_run(s, labels2, masks2, clusters2))
    for w, gg in zip(want, got):
        assert (w == gg).all()
    g.reset()


def test_non_default_stream(checker):
    from fast_slic_b200 import Slic
    K, B, H, W = 200, 4, 180, 250
    s = Slic(num_components=K, min_size_factor=0.1)
    imgs = torch.from_numpy(np.stack([make_image("syn", H, W, seed=60 + b) for b in range(B)])).cuda()
    masks = torch.from_numpy(np.random.RandomState(61).randint(0, 256, (B, H, W)).astype(np.uint8)).cuda()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        labels, clusters = s.iterate_batch(imgs, return_clusters=True)
        outs = _run(s, labels, masks, clusters)
    st.synchronize()
    _check(checker, K, labels, masks, clusters, outs)


def test_numpy_and_tensors_agree(superpixels):
    s, labels, masks, clusters = superpixels
    want = _host(_run(s, labels, masks, clusters))
    outs = _run(s, labels.cpu().numpy(), masks.cpu().numpy(), _struct(clusters))
    assert all(isinstance(x, np.ndarray) for x in outs)
    for w, g in zip(want, outs):
        assert w.dtype == g.dtype and (w == g).all()
