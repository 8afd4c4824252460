"""Episode replay buffer + proportional PER, restated in NumPy (oracle; test infra only).

Follows /root/reference/offpolicy/utils/rec_buffer.py and utils/segment_tree.py:
  * storage + ring insert      rec_buffer.py:85-141, 146-190
  * uniform sampling           rec_buffer.py:62-82, 192-240   (np.random.choice, with replacement)
  * reward normalisation       rec_buffer.py:209-223          (nan-masked mean / population std over ALL filled rewards)
  * PER trees, sampling, IS    rec_buffer.py:243-304, segment_tree.py:58-146
  * priority write-back        rec_buffer.py:306-324          (duplicate index: last write wins)

Output layout is the reference's: obs (N, T+1, B, O), share_obs (T+1, B, S) [same-share],
acts (N, T, B, A), rewards/dones (N, T, B, 1), dones_env (T, B, 1), avail (N, T+1, B, A).

Known reference defect restated as *intent* (SURVEY.md App. D-2): the reference's PER
`insert` loops `range(idx_range[0], idx_range[1])` and so never primes the new leaves;
here `prime_leaves=True` sets leaf = max_priority**alpha for every inserted slot.
"""
import numpy as np


def _to_agent_major(x):
    # (T, B, N, D) -> (N, T, B, D)  (rec_buffer.py:6-7)
    return x.transpose(2, 0, 1, 3)


class EpisodeStore(object):
    """One policy's SoA, time-major like the reference (rec_buffer.py:120-141)."""

    def __init__(self, capacity, T, N, O, S, A, same_share=True, use_avail=True, reward_norm=False):
        self.capacity, self.T, self.N = capacity, T, N
        self.same_share, self.use_avail, self.reward_norm = same_share, use_avail, reward_norm
        f32 = np.float32
        self.obs = np.zeros((T + 1, capacity, N, O), f32)
        self.share_obs = np.zeros((T + 1, capacity, S) if same_share else (T + 1, capacity, N, S), f32)
        self.acts = np.zeros((T, capacity, N, A), f32)
        self.avail = np.ones((T + 1, capacity, N, A), f32) if use_avail else None
        self.rewards = np.zeros((T, capacity, N, 1), f32)
        self.dones = np.ones((T, capacity, N, 1), f32)          # padding == done
        self.dones_env = np.ones((T, capacity, 1), f32)
        self.filled = 0
        self.cursor = 0

    def __len__(self):
        return self.filled

    def insert(self, n_ep, obs, share_obs, acts, rewards, dones, dones_env, avail=None):
        assert acts.shape[0] == self.T, "different dimension!"
        slots = (self.cursor + np.arange(n_ep)) % self.capacity       # ring with wrap (rec_buffer.py:167-171)
        if self.same_share:
            share_obs = share_obs[:, :, 0]
        self.obs[:, slots] = obs
        self.share_obs[:, slots] = share_obs
        self.acts[:, slots] = acts
        self.rewards[:, slots] = rewards
        self.dones[:, slots] = dones
        self.dones_env[:, slots] = dones_env
        if self.use_avail:
            self.avail[:, slots] = avail
        self.cursor = int(slots[-1]) + 1
        self.filled = min(self.filled + n_ep, self.capacity)
        return slots

    def reward_stats(self):
        """nan-masked mean/std over every filled reward (rec_buffer.py:209-220)."""
        de = self.dones_env[:, :self.filled]                              # (T, F, 1)
        prev_done = np.concatenate([np.zeros_like(de[:1]), de[:-1]], 0)    # shifted by one step
        mask = np.repeat(prev_done[:, :, None, :], self.N, axis=2) == 1.0
        r = self.rewards[:, :self.filled].copy()
        r[mask] = np.nan
        return np.nanmean(r), np.nanstd(r)

    def gather(self, inds):
        inds = np.asarray(inds)
        obs = _to_agent_major(self.obs[:, inds])
        acts = _to_agent_major(self.acts[:, inds])
        if self.reward_norm:
            mean, std = self.reward_stats()
            rewards = _to_agent_major((self.rewards[:, inds] - mean) / std)
        else:
            rewards = _to_agent_major(self.rewards[:, inds])
        share = self.share_obs[:, inds] if self.same_share else _to_agent_major(self.share_obs[:, inds])
        dones = _to_agent_major(self.dones[:, inds])
        dones_env = self.dones_env[:, inds]
        avail = _to_agent_major(self.avail[:, inds]) if self.use_avail else None
        return obs, share, acts, rewards, dones, dones_env, avail


class SegTree(object):
    """float64 array-backed tree, leaf i at cap+i (segment_tree.py:38, 74-94)."""

    def __init__(self, cap, op, neutral):
        assert cap > 0 and cap & (cap - 1) == 0
        self.cap, self.op = cap, op
        self.v = np.full(2 * cap, neutral, dtype=np.float64)

    def set(self, idx, val):
        idx = np.atleast_1d(np.asarray(idx, dtype=np.int64))
        val = np.broadcast_to(np.asarray(val, dtype=np.float64), idx.shape)
        self.v[idx + self.cap] = val                 # numpy fancy assign: last duplicate wins
        nodes = np.unique((idx + self.cap) // 2)
        while nodes.size and nodes[0] > 0:
            self.v[nodes] = self.op(self.v[2 * nodes], self.v[2 * nodes + 1])
            nodes = np.unique(nodes // 2)
            if nodes.size == 1 and nodes[0] == 0:
                break

    def get(self, idx):
        return self.v[self.cap + np.asarray(idx)]

    def reduce(self, start=0, end=None):
        """op over leaves [start, end) with the reference's recursion order (segment_tree.py:43-72)."""
        if end is None:
            end = self.cap
        if end < 0:
            end += self.cap
        end -= 1

        def rec(s, e, node, ns, ne):
            if s == ns and e == ne:
                return self.v[node]
            mid = (ns + ne) // 2
            if e <= mid:
                return rec(s, e, 2 * node, ns, mid)
            if mid + 1 <= s:
                return rec(s, e, 2 * node + 1, mid + 1, ne)
            return self.op(rec(s, mid, 2 * node, ns, mid), rec(mid + 1, e, 2 * node + 1, mid + 1, ne))

        return rec(start, end, 1, 0, self.cap - 1)

    def find_prefixsum(self, mass):
        """Root->leaf descent; `value[left] <= mass` goes right (segment_tree.py:130-146).  All masses descend together, one tree level
        per step: the same comparisons and subtractions, in the same order, as one descent per mass."""
        m = np.array(mass, dtype=np.float64).reshape(-1)
        node = np.ones(m.shape, dtype=np.int64)
        while node.size and node[0] < self.cap:      # every leaf is at the same depth
            lv = self.v[2 * node]
            right = lv <= m
            m = np.where(right, m - lv, m)
            node = 2 * node + right
        return (node - self.cap).reshape(np.shape(mass))


class UniformReplay(object):
    """RecReplayBuffer (rec_buffer.py:10-82) for a single shared policy 'policy_0'."""

    def __init__(self, capacity, T, N, O, S, A, same_share=True, use_avail=True, reward_norm=False, rng=None):
        self.store = EpisodeStore(capacity, T, N, O, S, A, same_share, use_avail, reward_norm)
        self.rng = rng  # LegacyMT19937 or None -> numpy global stream

    def __len__(self):
        return len(self.store)

    def insert(self, n_ep, *fields):
        return self.store.insert(n_ep, *fields)

    def draw(self, B):
        if self.rng is None:
            return np.random.choice(len(self), B)
        return self.rng.choice(len(self), B)

    def sample(self, B):
        inds = self.draw(B)
        return self.store.gather(inds) + (None, None), inds


class PrioritizedReplay(UniformReplay):
    """PrioritizedRecReplayBuffer (rec_buffer.py:243-324)."""

    def __init__(self, alpha, capacity, *a, prime_leaves=True, **kw):
        super().__init__(capacity, *a, **kw)
        self.alpha = alpha
        cap = 1
        while cap < capacity:
            cap *= 2
        self.sum_tree = SegTree(cap, np.add, 0.0)
        self.min_tree = SegTree(cap, np.minimum, float("inf"))
        self.max_priority = 1.0
        self.prime_leaves = prime_leaves

    def insert(self, n_ep, *fields):
        slots = self.store.insert(n_ep, *fields)
        if self.prime_leaves:      # intent of rec_buffer.py:263-268 (see module docstring)
            p = self.max_priority ** self.alpha
            self.sum_tree.set(slots, p)
            self.min_tree.set(slots, p)
        return slots

    def draw_mass(self, B):
        u = np.random.random(size=B) if self.rng is None else self.rng.random(B)
        total = self.sum_tree.reduce(0, len(self) - 1)     # exclusive end: newest leaf excluded (rec_buffer.py:273)
        return u * total

    def sample(self, B, beta):
        assert len(self) > B
        assert beta > 0
        inds = self.sum_tree.find_prefixsum(self.draw_mass(B))
        total = self.sum_tree.reduce()
        p_min = self.min_tree.reduce() / total
        max_w = (p_min * len(self)) ** (-beta)
        w = (self.sum_tree.get(inds) / total * len(self)) ** (-beta) / max_w
        return self.store.gather(inds) + (w, inds), inds

    def update_priorities(self, idx, prio):
        idx = np.asarray(idx)
        prio = np.asarray(prio)
        assert len(idx) == len(prio) and prio.min() > 0 and idx.min() >= 0 and idx.max() < len(self)
        leaf = prio ** self.alpha          # computed in the dtype handed in (fp32 from the trainer)
        self.sum_tree.set(idx, leaf)
        self.min_tree.set(idx, leaf)
        self.max_priority = max(self.max_priority, float(prio.max()))
