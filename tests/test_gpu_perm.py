"""GPU parity of ``pqn_permutation`` (csrc/pqn_perm.cu) with the oracle's restatement of ``jax.random.permutation``
(rounds of a stable sort by fresh 32-bit keys; purejaxql/pqn_minatar.py:299-321): bit-exact index permutations for
both threefry layouts, ragged sizes, the minibatch output layout, the oversized-bucket fallback and the full
BASELINE size (property checks).

jax runs ceil(3 ln n / ln(2^32 - 1)) rounds: none at n = 1, one up to n = 1,625, two up to 2,642,245 and three from
2,642,246 on.  The sizes below sit on both sides of each boundary, so a round count rounded the other way changes the
whole permutation, and 4,194,304 (65,536 Acrobot envs x 64 steps, BASELINE configs[3]) runs the third round, which
reads the ping buffer and writes ``out`` a second time."""
import numpy as np
import pytest
import torch

from oracle import jax_prng as jr

pytestmark = pytest.mark.gpu


def tkeys(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32).copy()).to("cuda:0")


@pytest.mark.parametrize("part", [0, 1])
@pytest.mark.parametrize("n", [1, 2, 37, 64, 65, 1000, 4096, 20000, 1625, 1626, 2642245, 2642246, 4194304])
def test_permutation_matches_oracle_bit_exact(n, part):
    """All three keys' permutations equal the oracle's.  Above a million elements the NumPy oracle takes seconds per
    key, so there only the last key (the largest seed offset) is compared; the smaller sizes cover the others."""
    from purejaxql_b200 import jaxrandom
    keys = np.stack([jr.PRNGKey(s) for s in (0, 5, 77)])
    got = jaxrandom.permutation_indices(tkeys(keys), n, part).cpu().numpy()
    assert got.shape == (3, n) and got.dtype == np.int32
    jr.DEFAULT_PARTITIONABLE = bool(part)
    try:
        for i in range(3) if n < 1_000_000 else [2]:
            assert np.array_equal(got[i], jr.permutation_indices(keys[i], n)), (n, part, i)
    finally:
        jr.DEFAULT_PARTITIONABLE = False


def _check_minibatch_layout(n, chunk):
    """The [n / chunk][S][chunk] minibatch layout is the plain [S][n] output transposed, and calls that reuse the
    workspace give the same results again."""
    from purejaxql_b200 import jaxrandom
    keys = np.stack([jr.PRNGKey(s) for s in (3, 4)])
    ws = jaxrandom.permutation_workspace(n, 2, "cuda:0")
    plain = jaxrandom.permutation_indices(tkeys(keys), n, 0, workspace=ws)
    mb = jaxrandom.permutation_indices(tkeys(keys), n, 0, chunk=chunk, workspace=ws)
    assert mb.shape == (n // chunk, 2, chunk)
    assert torch.equal(mb, plain.view(2, n // chunk, chunk).transpose(0, 1).contiguous())
    assert torch.equal(mb, jaxrandom.permutation_indices(tkeys(keys), n, 0, chunk=chunk, workspace=ws))
    assert torch.equal(plain, jaxrandom.permutation_indices(tkeys(keys), n, 0, workspace=ws))   # scratch state is reset


def test_permutation_minibatch_layout_and_workspace_reuse():
    _check_minibatch_layout(2048, 256)


def test_permutation_minibatch_layout_three_rounds():
    """BASELINE configs[3]: 4,194,304 samples per seed in the 16 minibatches of pqn_cartpole.yaml.  Three rounds run,
    and only the last may write the chunked layout: the second round's output is the third round's input."""
    _check_minibatch_layout(4194304, 262144)


def test_permutation_oversized_bucket_path():
    """Buckets of ~1024 elements (> the 256 a warp stages in shared memory) take the global-memory rank path."""
    from purejaxql_b200 import _lib, jaxrandom
    keys = np.stack([jr.PRNGKey(11)])
    prev = _lib.lib().pqn_set_permutation_bucket_log2(10)
    try:
        got = jaxrandom.permutation_indices(tkeys(keys), 8192, 0).cpu().numpy()
    finally:
        _lib.lib().pqn_set_permutation_bucket_log2(prev)
    assert np.array_equal(got[0], jr.permutation_indices(keys[0], 8192))


def test_permutation_full_size_properties():
    """BASELINE geometry (128 seeds x 131,072 samples): every row is a permutation, rows differ, seed 0 and seed 127
    equal the oracle."""
    from purejaxql_b200 import jaxrandom
    S, n = 128, 131072
    keys = jr.split(jr.PRNGKey(9), S)
    got = jaxrandom.permutation_indices(tkeys(keys), n, 0)
    srt = torch.sort(got, dim=1).values
    assert torch.equal(srt, torch.arange(n, device=got.device, dtype=torch.int32).expand(S, n))
    assert not torch.equal(got[0], got[1])
    g = got.cpu().numpy()
    for s in (0, 127):
        assert np.array_equal(g[s], jr.permutation_indices(keys[s], n))
