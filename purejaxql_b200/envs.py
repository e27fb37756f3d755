"""Host-side mirror of the gymnax environment protocol over libpqn_b200's
batched environment operator.

Mirrors what the reference uses of gymnax (purejaxql/pqn_minatar.py:103-112):

    env, env_params = make("Breakout-MinAtar")       # gymnax.make + LogWrapper
    obs, state = env.reset(keys, env_params)          # keys: uint32[N,2] (already split)
    obs, state, reward, done, info = env.step(keys, state, action, env_params)
    env.action_space(env_params).n, env.observation_space(env_params).shape,
    env_params.max_steps_in_episode

The functional protocol is kept (state in, state out) but batched natively —
there is no ``jax.vmap`` to wrap it with — and ``state`` is the library's
word-major SoA block (``uint32[state_words, N]`` CUDA tensor).
``state_to_fields`` / ``fields_to_state`` convert to and from gymnax's field
names for interop and parity tests (pure tensor ops, usable on CPU tensors).
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace

import torch

from . import _lib

ENV_IDS = {
    "Breakout-MinAtar": 0,
    "Asterix-MinAtar": 1,
    "SpaceInvaders-MinAtar": 2,
    "Freeway-MinAtar": 3,
    "Seaquest-MinAtar": 4,
    "CartPole-v1": 16,
    "Acrobot-v1": 17,
    "MountainCar-v0": 18,
    "MemoryChain-bsuite": 32,
    "Catch-bsuite": 33,
    "DeepSea-bsuite": 34,
    "UmbrellaChain-bsuite": 35,
    "DiscountingChain-bsuite": 36,
    "SimpleBandit-bsuite": 37,
    "BernoulliBandit-misc": 48,
    "FourRooms-misc": 49,
    "MetaMaze-misc": 50,
    "GaussianBandit-misc": 51,
}
# float-observation envs whose gymnax observation is 2-D although pqn_env_info's (rows, cols) = (1, 1) cannot say so
_2D_OBS = {"SimpleBandit-bsuite"}
# the MinAtar games gymnax 0.0.6 (the reference's pin) registers in gymnax.make
MINATAR_GAMES = ("Breakout-MinAtar", "Asterix-MinAtar", "SpaceInvaders-MinAtar", "Freeway-MinAtar")
# MinAtar games built here that gymnax 0.0.6 does not register (DESIGN.md section 8): restated from MinAtar itself
MINATAR_UNREGISTERED = ("Seaquest-MinAtar",)
# Seaquest-MinAtar's lists (bullets, fish, subs, divers): (capacity, first state word, entry fields)
_SQ_LISTS = (("f_bullets", 2, 4, ("x", "y", "lr")), ("e_fish", 8, 5, ("x", "y", "lr", "move_timer")),
             ("e_subs", 8, 9, ("x", "y", "lr", "move_timer", "shot_timer")),
             ("e_bullets", 8, 13, ("x", "y", "lr")), ("divers", 4, 17, ("x", "y", "lr", "move_timer")))
_SQ_FIELD_BITS = {"x": (0, 15), "y": (4, 15), "lr": (8, 1), "move_timer": (9, 7), "shot_timer": (12, 15)}
_SQ_LEN_BITS = {"f_bullets": (0, 3), "e_fish": (2, 15), "e_subs": (6, 15), "e_bullets": (10, 15), "divers": (14, 7)}

LOG_FIELDS = ("episode_returns", "episode_lengths", "returned_episode_returns",
              "returned_episode_lengths", "timestep")


@dataclass
class EnvParams:
    max_steps_in_episode: int
    memory_length: int = 5          # MemoryChain-bsuite's EnvParams.memory_length (gymnax default); other envs ignore it

    def as_c(self) -> _lib.EnvParams:
        """The ``pqn_env_params_t`` of ``pqn_env_reset_params``."""
        return _lib.EnvParams(int(self.max_steps_in_episode), int(self.memory_length))


def _u2f(t):
    return t.contiguous().view(torch.float32)


def _f2u(t):
    return t.to(torch.float32).contiguous().view(torch.int32)


# --------------------------------------------------------------------------- #
# state <-> gymnax field conversion (int32 views of the uint32 words)
# --------------------------------------------------------------------------- #
def state_to_fields(env_name: str, state: torch.Tensor) -> dict:
    """uint32/int32[state_words, N] -> dict of gymnax EnvState + LogEnvState fields."""
    st = state.view(torch.int32) if state.dtype != torch.int32 else state
    f = {}
    if env_name == "Breakout-MinAtar":
        w = st[0]
        f["ball_y"] = w & 15
        f["ball_x"] = (w >> 4) & 15
        f["ball_dir"] = (w >> 8) & 3
        f["pos"] = (w >> 10) & 15
        f["last_y"] = (w >> 14) & 15
        f["last_x"] = (w >> 18) & 15
        f["strike"] = ((w >> 22) & 1).bool()
        f["terminal"] = ((w >> 23) & 1).bool()
        f["time"] = st[1]
        n = st.shape[1]
        p = torch.arange(100, device=st.device)
        words = st[2:6].to(torch.int64) & 0xFFFFFFFF                       # [4, N]
        bits = (words[p >> 5] >> (p & 31).unsqueeze(1)) & 1                # [100, N]
        f["brick_map"] = bits.t().reshape(n, 10, 10).to(torch.float32)
        core = 6
    elif env_name == "Freeway-MinAtar":
        w = st[0]
        f["pos"] = w & 15
        f["move_timer"] = (w >> 4) & 3
        f["terminal"] = ((w >> 6) & 1).bool()
        f["time"] = st[1]
        cars = []
        for c in range(8):
            v = (st[2 + c // 2] >> (16 * (c % 2))) & 0xFFFF
            cars.append(torch.stack([v & 15, torch.full_like(v, c + 1), (v >> 4) & 7, ((v >> 7) & 15) - 5], -1))
        f["cars"] = torch.stack(cars, 1)                                    # [N, 8, 4] = (x, y, timer, speed)
        core = 6
    elif env_name == "Asterix-MinAtar":
        w, w1 = st[0], st[1]
        f["player_x"] = w & 15
        f["player_y"] = (w >> 4) & 15
        f["spawn_speed"] = (w >> 8) & 15
        f["spawn_timer"] = (w >> 12) & 15
        f["move_speed"] = (w >> 16) & 7
        f["move_timer"] = (w >> 19) & 7
        f["shot_timer"] = (w >> 22) & 7
        f["terminal"] = ((w >> 25) & 1).bool()
        f["ramp_timer"] = (w1 & 255) - 1
        f["ramp_index"] = (w1 >> 8) & 255
        f["time"] = st[2]
        ents = []
        for e in range(8):
            v = (st[3 + e // 4] >> (8 * (e % 4))) & 255
            fill = (v >> 6) & 1
            ents.append(torch.stack([v & 15, fill * (e + 1), (v >> 4) & 1, (v >> 5) & 1, fill], -1))
        f["entities"] = torch.stack(ents, 1)                                # [N, 8, 5] = (x, y, lr, is_gold, filled)
        core = 5
    elif env_name == "SpaceInvaders-MinAtar":
        w = st[0]
        f["pos"] = w & 15
        f["alien_dir"] = ((w >> 4) & 1) * 2 - 1
        f["enemy_move_interval"] = (w >> 5) & 15
        f["alien_move_timer"] = (w >> 9) & 15
        f["alien_shot_timer"] = (w >> 13) & 15
        f["shot_timer"] = (w >> 17) & 7
        f["terminal"] = ((w >> 20) & 1).bool()
        f["ramp_index"] = (w >> 21) & 15
        f["time"] = st[1]
        n = st.shape[1]
        p = torch.arange(100, device=st.device)
        for name, base in (("alien_map", 2), ("f_bullet_map", 6), ("e_bullet_map", 10)):
            words = st[base:base + 4].to(torch.int64) & 0xFFFFFFFF
            bits = (words[p >> 5] >> (p & 31).unsqueeze(1)) & 1
            f[name] = bits.t().reshape(n, 10, 10).to(torch.int32)
        core = 14
    elif env_name == "Seaquest-MinAtar":
        w, w1, w2 = st[0], st[1], st[2]
        f["sub_x"] = w & 15
        f["sub_y"] = (w >> 4) & 15
        f["sub_or"] = ((w >> 8) & 1).bool()
        f["shot_timer"] = (w >> 9) & 7
        f["diver_count"] = (w >> 12) & 7
        f["surface"] = ((w >> 15) & 1).bool()
        f["terminal"] = ((w >> 16) & 1).bool()
        f["move_speed"] = (w >> 17) & 7
        f["ramp_index"] = (w >> 20) & 31
        f["oxygen"] = (w1 & 255) - 1
        f["e_spawn_speed"] = (w1 >> 8) & 31
        f["e_spawn_timer"] = (w1 >> 13) & 31
        f["d_spawn_timer"] = (w1 >> 18) & 63
        f["time"] = st[3]
        for name, cap, w0, fields in _SQ_LISTS:
            sh, m = _SQ_LEN_BITS[name]
            f["n_" + name] = (w2 >> sh) & m
            ents = []
            for k in range(cap):
                v = (st[w0 + k // 2] >> (16 * (k % 2))) & 0xFFFF
                ents.append(torch.stack([(v >> _SQ_FIELD_BITS[c][0]) & _SQ_FIELD_BITS[c][1] for c in fields], -1))
            f[name] = torch.stack(ents, 1)                                  # [N, capacity, fields], zero past n_<name>
        core = 19
    elif env_name == "CartPole-v1":
        for j, k in enumerate(("x", "x_dot", "theta", "theta_dot")):
            f[k] = _u2f(st[j])
        f["time"] = st[4]
        core = 5
    elif env_name == "Acrobot-v1":
        for j, k in enumerate(("joint_angle1", "joint_angle2", "velocity_1", "velocity_2")):
            f[k] = _u2f(st[j])
        f["time"] = st[4]
        core = 5
    elif env_name == "MountainCar-v0":
        f["position"] = _u2f(st[0])
        f["velocity"] = _u2f(st[1])
        f["time"] = st[2]
        core = 3
    elif env_name == "Catch-bsuite":
        w = st[0]
        f["ball_x"] = w & 15
        f["ball_y"] = (w >> 4) & 15
        f["paddle_x"] = (w >> 8) & 15
        f["paddle_y"] = (w >> 12) & 15
        f["prev_done"] = ((w >> 16) & 1).bool()
        f["time"] = st[1]
        core = 2
    elif env_name == "MemoryChain-bsuite":
        f["context"] = (st[0] != 0).unsqueeze(1)                           # [N, num_bits = 1]
        for j, k in enumerate(("query", "total_perfect", "total_regret", "time", "memory_length"), 1):
            f[k] = st[j]                                                    # memory_length: the EnvParams word
        core = 6
    elif env_name == "DeepSea-bsuite":
        w = st[0]
        f["row"] = w & 255
        f["column"] = (w >> 8) & 255
        f["bad_episode"] = ((w >> 16) & 1).bool()
        f["total_bad_episodes"] = st[1]
        f["denoised_return"] = st[2]
        f["optimal_return"] = _u2f(st[3])
        f["optimal_no_cost"] = _u2f(st[4])
        n = st.shape[1]
        p = torch.arange(64, device=st.device)
        words = st[5:7].to(torch.int64) & 0xFFFFFFFF                       # [2, N]
        bits = (words[p >> 5] >> (p & 31).unsqueeze(1)) & 1                # [64, N]
        f["action_mapping"] = bits.t().reshape(n, 8, 8).to(torch.float32)
        f["time"] = st[7]
        core = 8
    elif env_name == "UmbrellaChain-bsuite":
        for j, k in enumerate(("need_umbrella", "has_umbrella", "total_regret", "time")):
            f[k] = st[j]
        core = 4
    elif env_name == "DiscountingChain-bsuite":
        # gymnax keeps the five rewards; the state keeps the index of the 1.1 among ones
        for j, k in enumerate(("context", "mapped_action", "time", "max_steps_in_episode")):
            f[k] = st[j]                                                    # max_steps_in_episode: the EnvParams word
        core = 4
    elif env_name == "SimpleBandit-bsuite":
        # gymnax keeps the eleven rewards; the state keeps action_mask, their indices into linspace(0, 1, 11)
        j = torch.arange(11, device=st.device)
        words = st[0:2].to(torch.int64) & 0xFFFFFFFF                       # [2, N]
        f["action_mask"] = ((words[j >> 3] >> (4 * (j & 7)).unsqueeze(1)) & 15).t().to(torch.int32)   # [N, 11]
        f["total_regret"] = _u2f(st[2])
        f["time"] = st[3]
        f["optimal_return"] = _u2f(st[4])                                   # the EnvParams word
        core = 5
    elif env_name == "BernoulliBandit-misc":
        f["last_action"] = st[0]
        f["last_reward"] = st[1]
        f["reward_probs"] = torch.stack([_u2f(st[2]), _u2f(st[3])], 1)     # [N, 2]
        f["exp_reward_best"] = _u2f(st[4])
        f["time"] = st[5]
        core = 6
    elif env_name == "FourRooms-misc":
        w = st[0]
        f["pos"] = torch.stack([w & 255, (w >> 8) & 255], 1)
        f["goal"] = torch.stack([(w >> 16) & 255, (w >> 24) & 255], 1)
        f["time"] = st[1]
        f["fail_prob"] = _u2f(st[2])                                        # the EnvParams word
        core = 3
    elif env_name == "MetaMaze-misc":
        f["last_action"] = st[0]
        f["last_reward"] = _u2f(st[1])
        w = st[2]
        f["pos"] = torch.stack([w & 255, (w >> 8) & 255], 1)
        f["goal"] = torch.stack([(w >> 16) & 255, (w >> 24) & 255], 1)
        f["time"] = st[3]
        f["reward"] = _u2f(st[4])                                           # the EnvParams word
        core = 5
    elif env_name == "GaussianBandit-misc":
        f["last_action"] = st[0]
        f["last_reward"] = _u2f(st[1])
        f["mu2"] = _u2f(st[2])
        f["exp_reward_best"] = _u2f(st[3])
        f["time"] = st[4]
        f["mu1"] = _u2f(st[5])                                              # the EnvParams words
        f["sigma_l"] = _u2f(st[6])
        core = 7
    else:
        raise KeyError(env_name)
    f["log_episode_returns"] = _u2f(st[core + 0])
    f["log_episode_lengths"] = st[core + 1]
    f["log_returned_episode_returns"] = _u2f(st[core + 2])
    f["log_returned_episode_lengths"] = st[core + 3]
    f["log_timestep"] = st[core + 4]
    return f


def fields_to_state(env_name: str, f: dict) -> torch.Tensor:
    """Inverse of :func:`state_to_fields` -> int32[state_words, N]."""
    i32 = lambda t: torch.as_tensor(t).to(torch.int32)
    if env_name == "Breakout-MinAtar":
        w = (i32(f["ball_y"]) | (i32(f["ball_x"]) << 4) | (i32(f["ball_dir"]) << 8) | (i32(f["pos"]) << 10)
             | (i32(f["last_y"]) << 14) | (i32(f["last_x"]) << 18) | (i32(f["strike"]) << 22)
             | (i32(f["terminal"]) << 23))
        n = w.shape[0]
        bm = (torch.as_tensor(f["brick_map"]).reshape(n, 100) != 0).to(torch.int64)
        words = []
        for k in range(4):
            lo, hi = 32 * k, min(100, 32 * k + 32)
            sh = torch.arange(hi - lo, device=bm.device)
            v = (bm[:, lo:hi] << sh).sum(1)
            v = torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32)
            words.append(v)
        core = [w, i32(f["time"])] + words
    elif env_name == "Freeway-MinAtar":
        cars = i32(f["cars"])
        words = []
        for k in range(4):
            v = torch.zeros_like(cars[:, 0, 0])
            for h in range(2):
                c = 2 * k + h
                v = v | ((cars[:, c, 0] | (cars[:, c, 2] << 4) | ((cars[:, c, 3] + 5) << 7)) << (16 * h))
            words.append(v)
        core = [i32(f["pos"]) | (i32(f["move_timer"]) << 4) | (i32(f["terminal"]) << 6), i32(f["time"])] + words
    elif env_name == "Asterix-MinAtar":
        ent = i32(f["entities"])
        w = (i32(f["player_x"]) | (i32(f["player_y"]) << 4) | (i32(f["spawn_speed"]) << 8) | (i32(f["spawn_timer"]) << 12)
             | (i32(f["move_speed"]) << 16) | (i32(f["move_timer"]) << 19) | (i32(f["shot_timer"]) << 22)
             | (i32(f["terminal"]) << 25))
        w1 = (i32(f["ramp_timer"]) + 1) | (i32(f["ramp_index"]) << 8)
        words = []
        for k in range(2):
            v = torch.zeros_like(w)
            for h in range(4):
                e = 4 * k + h
                b = (ent[:, e, 0] | (ent[:, e, 2] << 4) | (ent[:, e, 3] << 5) | (1 << 6)) * ent[:, e, 4]
                v = v | (b << (8 * h))
            words.append(v)
        core = [w, w1, i32(f["time"])] + words
    elif env_name == "SpaceInvaders-MinAtar":
        w = (i32(f["pos"]) | ((i32(f["alien_dir"]) > 0).to(torch.int32) << 4) | (i32(f["enemy_move_interval"]) << 5)
             | (i32(f["alien_move_timer"]) << 9) | (i32(f["alien_shot_timer"]) << 13) | (i32(f["shot_timer"]) << 17)
             | (i32(f["terminal"]) << 20) | (i32(f["ramp_index"]) << 21))
        n = w.shape[0]
        core = [w, i32(f["time"])]
        for name in ("alien_map", "f_bullet_map", "e_bullet_map"):
            bm = (torch.as_tensor(f[name]).reshape(n, 100) != 0).to(torch.int64)
            for k in range(4):
                lo, hi = 32 * k, min(100, 32 * k + 32)
                sh = torch.arange(hi - lo, device=bm.device)
                v = (bm[:, lo:hi] << sh).sum(1)
                core.append(torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32))
    elif env_name == "Seaquest-MinAtar":
        w = (i32(f["sub_x"]) | (i32(f["sub_y"]) << 4) | (i32(f["sub_or"]) << 8) | (i32(f["shot_timer"]) << 9)
             | (i32(f["diver_count"]) << 12) | (i32(f["surface"]) << 15) | (i32(f["terminal"]) << 16)
             | (i32(f["move_speed"]) << 17) | (i32(f["ramp_index"]) << 20))
        w1 = ((i32(f["oxygen"]) + 1) | (i32(f["e_spawn_speed"]) << 8) | (i32(f["e_spawn_timer"]) << 13)
              | (i32(f["d_spawn_timer"]) << 18))
        w2 = torch.zeros_like(w)
        words = []
        for name, cap, _, fields in _SQ_LISTS:
            w2 = w2 | (i32(f["n_" + name]) << _SQ_LEN_BITS[name][0])
            ent = i32(f[name])
            for k in range(0, cap, 2):
                v = torch.zeros_like(w)
                for h in range(2):
                    for j, c in enumerate(fields):
                        v = v | (ent[:, k + h, j] << (_SQ_FIELD_BITS[c][0] + 16 * h))
                words.append(v)
        core = [w, w1, w2, i32(f["time"])] + words
    elif env_name == "CartPole-v1":
        core = [_f2u(torch.as_tensor(f[k])) for k in ("x", "x_dot", "theta", "theta_dot")] + [i32(f["time"])]
    elif env_name == "Acrobot-v1":
        core = [_f2u(torch.as_tensor(f[k])) for k in
                ("joint_angle1", "joint_angle2", "velocity_1", "velocity_2")] + [i32(f["time"])]
    elif env_name == "MountainCar-v0":
        core = [_f2u(torch.as_tensor(f[k])) for k in ("position", "velocity")] + [i32(f["time"])]
    elif env_name == "Catch-bsuite":
        core = [i32(f["ball_x"]) | (i32(f["ball_y"]) << 4) | (i32(f["paddle_x"]) << 8) | (i32(f["paddle_y"]) << 12)
                | (i32(f["prev_done"]) << 16), i32(f["time"])]
    elif env_name == "MemoryChain-bsuite":
        ctx = i32(f["context"])
        core = [ctx.reshape(ctx.shape[0], -1)[:, 0]] + [i32(f[k]) for k in
                                                         ("query", "total_perfect", "total_regret", "time", "memory_length")]
    elif env_name == "DeepSea-bsuite":
        n = i32(f["row"]).shape[0]
        am = (torch.as_tensor(f["action_mapping"]).reshape(n, 64) != 0).to(torch.int64)
        sh = torch.arange(32, device=am.device)
        words = [(am[:, 32 * k:32 * k + 32] << sh).sum(1) for k in range(2)]
        words = [torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32) for v in words]
        core = [i32(f["row"]) | (i32(f["column"]) << 8) | (i32(f["bad_episode"]) << 16), i32(f["total_bad_episodes"]),
                i32(f["denoised_return"]), _f2u(torch.as_tensor(f["optimal_return"])),
                _f2u(torch.as_tensor(f["optimal_no_cost"]))] + words + [i32(f["time"])]
    elif env_name == "UmbrellaChain-bsuite":
        core = [i32(f[k]) for k in ("need_umbrella", "has_umbrella", "total_regret", "time")]
    elif env_name == "DiscountingChain-bsuite":
        core = [i32(f[k]) for k in ("context", "mapped_action", "time", "max_steps_in_episode")]
    elif env_name == "SimpleBandit-bsuite":
        m = torch.as_tensor(f["action_mask"]).to(torch.int64)                # [N, 11]
        sh = 4 * torch.arange(8, device=m.device)
        words = [(m[:, 0:8] << sh).sum(1), (m[:, 8:11] << sh[:3]).sum(1)]
        words = [torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32) for v in words]
        core = words + [_f2u(torch.as_tensor(f["total_regret"])), i32(f["time"]),
                        _f2u(torch.as_tensor(f["optimal_return"]))]
    elif env_name == "BernoulliBandit-misc":
        p = torch.as_tensor(f["reward_probs"])
        core = [i32(f["last_action"]), i32(f["last_reward"]), _f2u(p[:, 0]), _f2u(p[:, 1]),
                _f2u(torch.as_tensor(f["exp_reward_best"])), i32(f["time"])]
    elif env_name in ("FourRooms-misc", "MetaMaze-misc"):
        pos, goal = i32(f["pos"]), i32(f["goal"])
        w = pos[:, 0] | (pos[:, 1] << 8) | (goal[:, 0] << 16) | (goal[:, 1] << 24)
        if env_name == "FourRooms-misc":
            core = [w, i32(f["time"]), _f2u(torch.as_tensor(f["fail_prob"]))]
        else:
            core = [i32(f["last_action"]), _f2u(torch.as_tensor(f["last_reward"])), w, i32(f["time"]),
                    _f2u(torch.as_tensor(f["reward"]))]
    elif env_name == "GaussianBandit-misc":
        core = [i32(f["last_action"]), _f2u(torch.as_tensor(f["last_reward"])), _f2u(torch.as_tensor(f["mu2"])),
                _f2u(torch.as_tensor(f["exp_reward_best"])), i32(f["time"]), _f2u(torch.as_tensor(f["mu1"])),
                _f2u(torch.as_tensor(f["sigma_l"]))]
    else:
        raise KeyError(env_name)
    log =[_f2u(torch.as_tensor(f["log_episode_returns"])), i32(f["log_episode_lengths"]),
           _f2u(torch.as_tensor(f["log_returned_episode_returns"])), i32(f["log_returned_episode_lengths"]),
           i32(f["log_timestep"])]
    return torch.stack(core + log).contiguous()


def pack_observation(obs: torch.Tensor) -> torch.Tensor:
    """{0,1} observations [N, ...] (e.g. the float32 (10,10,C) rows gymnax returns) ->
    int32[N, packed_obs_words] rows in the bit layout the CNN kernels read
    (bit f of a row = element f of the flattened observation; rows padded to 16 bytes)."""
    n = obs.shape[0]
    flat = (obs.reshape(n, -1) != 0).to(torch.int64)
    nb = flat.shape[1]
    pw = ((nb + 31) // 32 + 3) // 4 * 4
    padded = torch.zeros((n, pw * 32), dtype=torch.int64, device=obs.device)
    padded[:, :nb] = flat
    sh = torch.arange(32, device=obs.device, dtype=torch.int64)
    words = (padded.view(n, pw, 32) << sh).sum(-1)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
    return words.to(torch.int32).contiguous()


def reset_into(env_id: int, keys: torch.Tensor, state: torch.Tensor, obs: torch.Tensor | None, n: int,
               params: EnvParams, rng_mode: int):
    """``pqn_env_reset_params``: reset n envs into ``state`` (and ``obs`` unless None) with ``params``.  Parameters
    other than max_steps stay in the state block, so steps and auto-resets need nothing more."""
    _lib.check(_lib.lib().pqn_env_reset_params(env_id, _lib.p(keys), _lib.p(state), _lib.p(obs), n, params.as_c(),
                                               rng_mode, _lib.stream_ptr()), "pqn_env_reset_params")


def check_name(name: str):
    """Refuse a name that is not an env of ``ENV_IDS`` (host-side: builds nothing)."""
    if name not in ENV_IDS:
        raise KeyError(f"unknown env {name!r}; known: {sorted(ENV_IDS)}")


# --------------------------------------------------------------------------- #
# the batched environment
# --------------------------------------------------------------------------- #
class BatchedEnv:
    """``LogWrapper(gymnax.make(name)[0])`` (optionally with
    ``FlattenObservationWrapper``), batched over the leading axis."""

    def __init__(self, name: str, flatten_obs: bool = False, rng_mode: int = 0):
        check_name(name)
        self.name = name
        self.env_id = ENV_IDS[name]
        info = _lib.EnvInfo()
        _lib.check(_lib.lib().pqn_env_info(self.env_id, info), "pqn_env_info")
        self.info = info
        self.state_words = info.state_words
        self.obs_dim = info.obs_dim
        self.binary_obs = bool(info.binary_obs)
        self.packed_obs_words = info.packed_obs_words
        self.num_actions = info.num_actions
        if self.binary_obs:
            shape = tuple(info.obs_shape)
        else:   # a vector, or a 2-D board (Catch-bsuite's (10, 5), DeepSea-bsuite's (8, 8), SimpleBandit-bsuite's
            # (1, 1)): gymnax's unflattened shape
            board = info.obs_shape[1] > 1 or name in _2D_OBS
            shape = (info.obs_shape[0], info.obs_shape[1]) if board else (info.obs_dim,)
        self._obs_shape = (info.obs_dim,) if flatten_obs else shape
        self.default_params = EnvParams(max_steps_in_episode=info.max_steps)
        self.rng_mode = rng_mode

    # gymnax spaces -------------------------------------------------------
    def action_space(self, params=None):
        return SimpleNamespace(n=self.num_actions)

    def observation_space(self, params=None):
        return SimpleNamespace(shape=self._obs_shape)

    # protocol ------------------------------------------------------------
    def reset(self, keys: torch.Tensor, params: EnvParams | None = None):
        params = params or self.default_params
        n = keys.shape[0]
        state = torch.empty((self.state_words, n), dtype=torch.int32, device=keys.device)
        obs = torch.empty((n,) + self._obs_shape, dtype=torch.float32, device=keys.device)
        reset_into(self.env_id, keys, state, obs, n, params, self.rng_mode)
        return obs, state

    def step(self, keys: torch.Tensor, state: torch.Tensor, action: torch.Tensor,
             params: EnvParams | None = None, inplace: bool = False):
        params = params or self.default_params
        n = keys.shape[0]
        dev = keys.device
        state = state if inplace else state.clone()
        obs = torch.empty((n,) + self._obs_shape, dtype=torch.float32, device=dev)
        reward = torch.empty(n, dtype=torch.float32, device=dev)
        done = torch.empty(n, dtype=torch.uint8, device=dev)
        disc = torch.empty(n, dtype=torch.float32, device=dev)
        ret = torch.empty(n, dtype=torch.float32, device=dev)
        ln = torch.empty(n, dtype=torch.int32, device=dev)
        ts = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(_lib.lib().pqn_env_step(
            self.env_id, _lib.p(keys), _lib.p(state), _lib.p(action.to(torch.int32).contiguous()), _lib.p(obs),
            _lib.p(reward), _lib.p(done), _lib.p(disc), _lib.p(ret), _lib.p(ln), _lib.p(ts), n,
            params.max_steps_in_episode, self.rng_mode, _lib.stream_ptr()), "pqn_env_step")
        done_b = done.bool()
        info = {"discount": disc, "returned_episode_returns": ret, "returned_episode_lengths": ln,
                "timestep": ts, "returned_episode": done_b}
        return obs, state, reward, done_b, info


def make(env_name: str, flatten_obs: bool = False, rng_mode: int = 0):
    """``gymnax.make(env_name)`` -> (env, env_params); the LogWrapper is built in."""
    env = BatchedEnv(env_name, flatten_obs=flatten_obs, rng_mode=rng_mode)
    return env, env.default_params
