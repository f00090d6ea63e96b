"""The database chunk plan of the K-best list kernels (list_plan in match_kernels.cu): the chunks the planted triangulation scenes
and the key-frame search's scratch figures assume, and an empty database, which the plan gives one empty chunk, so that
hamming_topk returns the "no entry" lists."""
import numpy as np
import pytest

import triangulation_model as tm


def test_chunk_plan_of_the_scenes():
    """chunk_of restates list_plan; on a 132-SM H100 the "ties" scene (capacity 312) cuts its camera's database at row 256, between
    its tied candidates 251 .. 260, and the "capacity" scene (65535) puts rows 65468 and 65534 in the last of three chunks"""
    assert tm.H100_SMS == 132
    assert tm.chunk_of(312, 3) == (256, 2)
    assert tm.chunk_of(65535, 3) == (22016, 3) and 2 * 22016 <= 65468
    # the key-frame search's plan has the same form: on a config-3 frame (NS = 8000), 32 chunks for one candidate, 5 for 16
    assert tm.chunk_of(8000, 1) == (256, 32)
    assert tm.chunk_of(8000, 16) == (1792, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 32, 64])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("K", [1, 4, 8])
def test_hamming_topk_empty_database(api, dim, masked, K):
    """nd == 0: every query's list is K entries of index -1 and distance INT_MAX, from the host and the device entry points"""
    import torch
    rng = np.random.default_rng(100 * dim + 10 * masked + K)
    nq = 300
    q = rng.integers(0, 256, (nq, dim), dtype=np.uint8)
    qm = rng.integers(0, 256, (nq, dim), dtype=np.uint8) if masked else None
    d = np.zeros((0, dim), np.uint8)
    dm = np.zeros((0, dim), np.uint8) if masked else None
    want_i, want_d = np.full((nq, K), -1, np.int32), np.full((nq, K), 2**31 - 1, np.int32)
    idx, dist = api.hamming_topk(q, d, K, qm, dm)
    assert np.array_equal(idx, want_i) and np.array_equal(dist, want_d)
    dev = torch.device("cuda", 0)
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)  # noqa: E731
    # nd = 0 at a valid database address: a NULL one is refused, and torch gives an empty tensor none
    d_t = torch.zeros((1, dim), dtype=torch.uint8, device=dev)
    dm_t = torch.zeros((1, dim), dtype=torch.uint8, device=dev) if masked else None
    q_t, qm_t = t(q), t(qm)
    gi, gd = (torch.zeros((nq, K), dtype=torch.int32, device=dev) for _ in range(2))
    api._check(api.lib().mcs_hamming_topk_device(api._dptr(q_t), api._dptr(qm_t), nq, api._dptr(d_t), api._dptr(dm_t), 0, None, dim, K,
                                                 api._dptr(gi), api._dptr(gd), None))
    torch.cuda.synchronize(dev)
    assert np.array_equal(gi.cpu().numpy(), want_i) and np.array_equal(gd.cpu().numpy(), want_d)
