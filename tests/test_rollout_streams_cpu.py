"""Properties of the rollout's Philox convention (include/rcmarl.h, rcmarl_rollout) on its restatement
(tests/rollout_oracle.py), without a GPU: uniform resets over every grid shape, 24-bit action uniforms that are
independent of each other and across steps, agents, environments and episodes, the mu-mixture of get_action, and
counter sets of the reset, action and attack streams that never meet.  Every draw comes from a fixed seed, so every
check is deterministic; the chi-square tests use a significance of 1e-4."""
import numpy as np
import pytest
from scipy import stats

import rollout_oracle as R
from attack_oracle import counter as attack_counter
from oracle import rpbcac_oracle as O

SEED = 0x5EED0000BEEF
ALPHA = 1e-4


def draws(n_envs=512, n_episodes=4, max_ep_len=6, n_slots=5, n_active=5, nrow=5, ncol=5, seed=SEED, env_offset=0,
          episode_offset=0):
    return R.rollout_draws(seed, env_offset=env_offset, n_envs=n_envs, episode_offset=episode_offset,
                           n_episodes=n_episodes, max_ep_len=max_ep_len, n_slots=n_slots, n_active=n_active, nrow=nrow,
                           ncol=ncol)


def chi2_uniform(counts):
    counts = np.asarray(counts, np.float64).reshape(-1)
    return stats.chisquare(counts).pvalue


def chi2_independent(a, b, na, nb):
    """Chi-square test of independence of two discrete samples with values in [0, na) x [0, nb)."""
    table = np.zeros((na, nb))
    np.add.at(table, (np.asarray(a).reshape(-1), np.asarray(b).reshape(-1)), 1)
    return stats.chi2_contingency(table, correction=False).pvalue


def bins(u, k=10):
    return np.minimum((np.asarray(u, np.float64) * k).astype(np.int64), k - 1)


# ------------------------------------------------------------------------------------------------------------- resets
@pytest.mark.parametrize("nrow,ncol", [(1, 1), (5, 5), (4, 6), (6, 4), (3, 7), (10, 10), (32, 32)])
def test_resets_uniform_over_the_grid(nrow, ncol):
    """px = umulhi(x, nrow), py = umulhi(y, ncol): every cell of nrow x ncol equally likely, nothing outside it."""
    n_envs = max(2048, 24 * nrow * ncol)
    init, _ = draws(n_envs=n_envs, n_episodes=2, max_ep_len=1, nrow=nrow, ncol=ncol)
    x, y = init[..., 0], init[..., 1]
    assert x.min() >= 0 and x.max() < nrow and y.min() >= 0 and y.max() < ncol
    if nrow * ncol == 1:
        assert not x.any() and not y.any()
        return
    counts = np.bincount((x * ncol + y).reshape(-1), minlength=nrow * ncol)
    assert counts.min() > 0
    assert chi2_uniform(counts) > ALPHA
    if nrow > 1:
        assert chi2_uniform(np.bincount(x.reshape(-1), minlength=nrow)) > ALPHA
    if ncol > 1:
        assert chi2_uniform(np.bincount(y.reshape(-1), minlength=ncol)) > ALPHA


@pytest.mark.parametrize("nrow,ncol", [(5, 5), (4, 6), (10, 10)])
def test_resets_independent_between_coordinates_and_agents(nrow, ncol):
    init, _ = draws(n_envs=4096, n_episodes=2, max_ep_len=1, nrow=nrow, ncol=ncol)
    x, y = init[..., 0], init[..., 1]
    assert chi2_independent(x, y, nrow, ncol) > ALPHA
    assert chi2_independent(x[..., 0], x[..., 1], nrow, nrow) > ALPHA
    assert chi2_independent(y[..., 0], y[..., 4], ncol, ncol) > ALPHA
    assert chi2_independent(x[..., 2], y[..., 3], nrow, ncol) > ALPHA
    assert chi2_independent(x[0], x[1], nrow, nrow) > ALPHA                 # consecutive episodes, same env and agent


def test_reset_depends_on_every_counter_word():
    """Changing the env (across the 2^32 boundary too), the episode or the seed's high word changes the draw."""
    base = draws(n_envs=64, n_episodes=2, max_ep_len=1, nrow=32, ncol=32, env_offset=2 ** 32 - 32)[0]
    for kw in (dict(env_offset=2 ** 32 - 31), dict(episode_offset=1), dict(seed=SEED ^ (1 << 40))):
        other = draws(n_envs=64, n_episodes=2, max_ep_len=1, nrow=32, ncol=32, **{"env_offset": 2 ** 32 - 32, **kw})[0]
        assert (other != base).mean() > 0.9


# ------------------------------------------------------------------------------------------------------------- uniforms
def test_uniforms_are_24_bit_and_in_unit_interval():
    _, u = draws(n_envs=256, n_episodes=3, max_ep_len=8, n_slots=16, n_active=7)
    assert u.dtype == np.float32 and u.shape == (3, 8, 256, 7, 3)
    assert u.min() >= 0.0 and u.max() < 1.0
    k = u.astype(np.float64) * 2.0 ** 24
    assert np.array_equal(k, np.floor(k))
    for c in range(3):
        assert chi2_uniform(np.bincount(bins(u[..., c], 50).reshape(-1), minlength=50)) > ALPHA


@pytest.mark.parametrize("a,b", [(0, 1), (0, 2), (1, 2)])
def test_uniforms_pairwise_independent_within_a_draw(a, b):
    _, u = draws(n_envs=1024)
    assert chi2_independent(bins(u[..., a]), bins(u[..., b]), 10, 10) > ALPHA


@pytest.mark.parametrize("axis", ["step", "agent", "env", "episode"])
def test_uniforms_independent_across_neighbouring_counters(axis):
    """u of (step j, agent i, env e, episode k) against the same component one step / agent / env / episode on:
    a 2-D chi-square per component and across components (u0 here against u2 there)."""
    _, u = draws(n_envs=1024, n_episodes=4, max_ep_len=6)
    sl = {"episode": (np.s_[:-1], np.s_[1:]), "step": (np.s_[:, :-1], np.s_[:, 1:]),
          "env": (np.s_[:, :, :-1], np.s_[:, :, 1:]), "agent": (np.s_[:, :, :, :-1], np.s_[:, :, :, 1:])}[axis]
    here, there = u[sl[0]], u[sl[1]]
    for a, b in ((0, 0), (1, 1), (2, 2), (0, 2), (2, 1)):
        assert chi2_independent(bins(here[..., a]), bins(there[..., b]), 10, 10) > ALPHA, (a, b)


def test_action_stride_is_the_instantiation_width():
    """A padded team (n_active < n_slots) draws the same uniforms for its agents as the full instantiation: the action
    counter is step * n_slots + agent, never step * n_active + agent."""
    _, full = draws(n_envs=32, n_slots=16, n_active=16, max_ep_len=5)
    _, part = draws(n_envs=32, n_slots=16, n_active=7, max_ep_len=5)
    assert np.array_equal(part, full[..., :7, :])
    _, dense = draws(n_envs=32, n_slots=7, n_active=7, max_ep_len=5)
    assert np.array_equal(dense[:, 0], part[:, 0]) and (dense[:, 1:] != part[:, 1:]).mean() > 0.9


@pytest.mark.parametrize("mu", [0.0, 0.1, 1.0])
def test_action_frequencies_follow_the_mixture(mu):
    """O.sample_action_from_uniforms on the restated uniforms with fixed probabilities pi: P(a) = (1 - mu) pi + mu / 5."""
    pi = np.array([0.05, 0.35, 0.1, 0.3, 0.2], np.float32)
    _, u = draws(n_envs=4096, n_episodes=2, max_ep_len=5)
    u = u.reshape(-1, 3)
    a = O.sample_action_from_uniforms(np.broadcast_to(pi, (u.shape[0], 5)), u, mu)
    counts = np.bincount(a, minlength=5)
    want = ((1.0 - mu) * pi.astype(np.float64) + mu / 5.0) * u.shape[0]
    assert stats.chisquare(counts, want).pvalue > ALPHA


# ------------------------------------------------------------------------------------------------------------- counters
def counter_set(words):
    w = [np.asarray(x, np.uint64).reshape(-1) for x in words]
    return set(zip(*[x.tolist() for x in w]))


def test_counter_words_of_the_three_streams_never_meet():
    """Word 1 alone keeps the streams apart for every shard a Trainer can own (env_offset = rank * N, N <= 8192,
    world <= 8) and across env_offset >= 2^32: reset counters have bit 31 set, action counters have it clear, attack
    counters have bit 31 clear and bit 30 set, and no env index below 2^62 reaches bit 30 of word 1."""
    attack_w1 = {(a | r << 8 | R.ATTACK_BIT) for a in range(256) for r in range(256)}
    assert {int(attack_counter(1, a, r, 0, 0)[1][0]) for a in (0, 255) for r in (0, 255)} <= attack_w1
    offsets = [rank * N for N in (1, 64, 4096, 8192) for rank in range(8)] + [2 ** 32 - 5, 2 ** 32 + 7, 2 ** 40, 2 ** 62 - 9]
    for off in offsets:
        kw = dict(env_offset=off, n_envs=9, episode_offset=0, n_episodes=1)
        reset_w1 = set(R.reset_counters(n_active=1, **kw)[1].reshape(-1).tolist())
        action_w1 = set(R.action_counters(max_ep_len=1, n_slots=5, n_active=1, **kw)[1].reshape(-1).tolist())
        assert all(w & R.RESET_BIT for w in reset_w1)
        assert not any(w & R.RESET_BIT for w in action_w1)
        assert not reset_w1 & action_w1 and not reset_w1 & attack_w1 and not action_w1 & attack_w1, off


@pytest.mark.parametrize("env_offset,n_envs,n_slots", [(0, 8192, 5), (7 * 8192, 8192, 16), (2 ** 32 - 40, 80, 16)])
def test_counter_sets_are_disjoint(env_offset, n_envs, n_slots):
    """The full 4-word counter sets of a block's reset and action draws and of an update round's attack draws, built
    element by element: no two draws of a block share a counter, and no counter is in two streams."""
    n_ep, L_ = 3, 4
    kw = dict(env_offset=env_offset, n_envs=n_envs, episode_offset=2 ** 32 - 2, n_episodes=n_ep)
    rc = counter_set(R.reset_counters(n_active=n_slots, **kw))
    ac = counter_set(R.action_counters(max_ep_len=L_, n_slots=n_slots, n_active=n_slots, **kw))
    assert len(rc) == n_ep * n_envs * n_slots and len(ac) == n_ep * L_ * n_envs * n_slots
    att = set()
    for a, r in ((4, 0), (255, 255), (0, 1)):
        att |= counter_set(attack_counter(2000, a, r, 2 ** 32 - 2, 1))
    assert not rc & ac and not rc & att and not ac & att


def test_episode_word_wraps_at_2_32():
    """The episode word is the low 32 bits of episode_offset + episode."""
    a = draws(n_envs=16, n_episodes=3, max_ep_len=2, episode_offset=2 ** 32 - 2)
    b = draws(n_envs=16, n_episodes=1, max_ep_len=2, episode_offset=0)
    c = draws(n_envs=16, n_episodes=1, max_ep_len=2, episode_offset=2 ** 33)
    for x, y, z in zip(a, b, c):
        assert np.array_equal(x[2], y[0]) and np.array_equal(y[0], z[0])
        assert not np.array_equal(x[0], x[2])
