"""Batched value-network robot policies on top of the fused lookahead kernel.

The networks themselves stay plain PyTorch on the same device (north_star: "SARL's attention net stays PyTorch"); what
is replaced is the reference's per-action Python loop (crowd_nav/policy/multi_human_rl.py:35-56, cadrl.py:156-170):
81 x [env.onestep_lookahead (N ORCA solves each) + propagate + 5 tiny H2D copies + rotate + model(...).item()] per
decision becomes ONE crowdsim_lookahead_pack launch (N ORCA solves per env, shared by all actions) + ONE batched
forward over [B*81][N][13] + an argmax on device.

Module / parameter names of the networks equal the reference's (sarl.py:9-65, cadrl.py:11-29), so reference
checkpoints (rl_model.pth / il_model.pth state_dicts) load unchanged with load_state_dict().
"""
import itertools
import logging

import numpy as np
import torch
import torch.nn as nn


def mlp(input_dim, mlp_dims, last_relu=False):
    """cadrl.py:11-19"""
    layers = []
    dims = [input_dim] + list(mlp_dims)
    for i in range(len(dims) - 1):
        layers.append(nn.Linear(dims[i], dims[i + 1]))
        if i != len(dims) - 2 or last_relu:
            layers.append(nn.ReLU())
    return nn.Sequential(*layers)


def build_action_space(v_pref, speed_samples=5, rotation_samples=16, kinematics='holonomic'):
    """cadrl.py:82-102 as an [A][2] float64 array: (0,0) first, then rotations x speeds (rotation-major)."""
    holonomic = kinematics == 'holonomic'
    speeds = [(np.exp((i + 1) / speed_samples) - 1) / (np.e - 1) * v_pref for i in range(speed_samples)]
    if holonomic:
        rotations = np.linspace(0, 2 * np.pi, rotation_samples, endpoint=False)
    else:
        rotations = np.linspace(-np.pi / 4, np.pi / 4, rotation_samples)
    space = [(0.0, 0.0)]
    for rotation, speed in itertools.product(rotations, speeds):
        if holonomic:
            space.append((speed * np.cos(rotation), speed * np.sin(rotation)))
        else:
            space.append((speed, rotation))
    return np.array(space, dtype=np.float64)


class CADRLValueNetwork(nn.Module):
    """cadrl.py:22-29 (parameter prefix `value_network.`)."""

    def __init__(self, input_dim=13, mlp_dims=(150, 100, 100, 1)):
        super().__init__()
        self.value_network = mlp(input_dim, mlp_dims)

    def forward(self, state):
        return self.value_network(state)


class SARLValueNetwork(nn.Module):
    """sarl.py:9-65. forward(state[batch][humans][13]) -> value[batch][1]. The reference copies the attention weights of
    sample 0 to the host on every forward (sarl.py:54, visualisation only); here they stay on device in
    `attention_weights` and are materialised on request."""

    def __init__(self, input_dim=13, self_state_dim=6, mlp1_dims=(150, 100), mlp2_dims=(100, 50),
                 mlp3_dims=(150, 100, 100, 1), attention_dims=(100, 100, 1), with_global_state=True):
        super().__init__()
        self.self_state_dim = self_state_dim
        self.global_state_dim = mlp1_dims[-1]
        self.mlp1 = mlp(input_dim, mlp1_dims, last_relu=True)
        self.mlp2 = mlp(mlp1_dims[-1], mlp2_dims)
        self.with_global_state = with_global_state
        self.attention = mlp(mlp1_dims[-1] * 2 if with_global_state else mlp1_dims[-1], attention_dims)
        self.mlp3 = mlp(mlp2_dims[-1] + self_state_dim, mlp3_dims)
        self.attention_weights = None

    def forward(self, state):
        b, n, d = state.shape
        self_state = state[:, 0, :self.self_state_dim]
        h1 = self.mlp1(state.reshape(b * n, d))
        h2 = self.mlp2(h1)
        if self.with_global_state:
            g = h1.view(b, n, -1).mean(dim=1, keepdim=True).expand(b, n, self.global_state_dim).reshape(b * n, -1)
            att_in = torch.cat([h1, g], dim=1)
        else:
            att_in = h1
        scores = self.attention(att_in).view(b, n)
        scores_exp = torch.exp(scores) * (scores != 0).float()          # sarl.py:52 "masked softmax"
        weights = (scores_exp / scores_exp.sum(dim=1, keepdim=True)).unsqueeze(2)
        self.attention_weights = weights[0, :, 0].detach()
        feat = (weights * h2.view(b, n, -1)).sum(dim=1)
        return self.mlp3(torch.cat([self_state, feat], dim=1))


class LSTMRLValueNetwork(nn.Module):
    """lstm_rl.py:9-65 (ValueNetwork1, or ValueNetwork2 when mlp1_dims is given = "with_interaction_module"): the humans'
    rows go through an LSTM in the order given, the final hidden state joins the robot's 6 features in an MLP.
    h0/c0 are created on the input's device (the reference creates them on the CPU, lstm_rl.py:27-28, which breaks
    under --gpu). With query_env=true the lookahead states reach the network in env order (SURVEY quirk 9)."""

    def __init__(self, input_dim=13, self_state_dim=6, mlp_dims=(150, 100, 100, 1), lstm_hidden_dim=50, mlp1_dims=None):
        super().__init__()
        self.self_state_dim = self_state_dim
        self.lstm_hidden_dim = lstm_hidden_dim
        if mlp1_dims is not None:
            self.mlp1 = mlp(input_dim, mlp1_dims)
        self.mlp = mlp(self_state_dim + lstm_hidden_dim, mlp_dims)
        self.lstm = nn.LSTM(mlp1_dims[-1] if mlp1_dims is not None else input_dim, lstm_hidden_dim, batch_first=True)
        self.has_mlp1 = mlp1_dims is not None

    def forward(self, state):
        b, n, d = state.shape
        self_state = state[:, 0, :self.self_state_dim]
        x = self.mlp1(state.reshape(b * n, d)).reshape(b, n, -1) if self.has_mlp1 else state
        h0 = torch.zeros(1, b, self.lstm_hidden_dim, device=state.device, dtype=state.dtype)
        _, (hn, _) = self.lstm(x, (h0, torch.zeros_like(h0)))
        return self.mlp(torch.cat([self_state, hn.squeeze(0)], dim=1))


class BatchedValuePolicy(object):
    """One-step-lookahead policy over a value network (MultiHumanRL.predict / CADRL.predict): greedy in the test / val
    phases, epsilon-greedy in the train phase (multi_human_rl.py:27-31, cadrl.py:148-152: with probability epsilon a
    uniformly drawn action of the 81-action space). The reference draws from numpy's GLOBAL generator (re-seeded by every
    env.reset, shared with scenario generation). exploration='torch' (default): every env has its own uniform draw from a
    torch.Generator on the policy's device (set_seed): same distribution, a different random stream -- RL-phase rollouts
    are statistically, not bitwise, reproductions of the reference's. exploration='numpy': the draws come from each env's
    copy of numpy's stream as the reference's reset leaves it (env.policy_draws, once per act_batch), so the exploring
    decisions are the reference's own; the env needs episode tracking.

    act_batch(env) -> [B][2] float64 device tensor with, per env,
        argmax_a  reward(s, a) + gamma ** (time_step * v_pref) * V(rotate(next_state(s, a)))       multi_human_rl.py:52
    or the zero action when the robot already is within its radius of the goal (policy.py:41-48).
    `joint` selects how humans enter the network: True = one [N][13] set per action (SARL, LSTM-RL, multi_human_rl.py:45),
    False = CADRL's min over per-human values (cadrl.py:163-166).
    query_env (policy.config [action_space]): True asks the simulator (env.onestep_lookahead: lookahead_pack, the humans' ORCA
    decisions and the env's reward); False extrapolates every human at its own velocity and uses the policy's compute_reward
    (multi_human_rl.py:38-42: propagate_pack). CADRL always queries the env (cadrl.py:156-170), so joint=False with
    query_env=False is refused. order_by_distance: with query_env=False the rows follow LSTM-RL's sort by decreasing
    distance to the robot (lstm_rl.py:99-103). sort_last_state: the policy's stored last_state (the rows of its replay
    pairs) has that sort too, with either query_env (LSTM-RL); lookahead rows with query_env=True stay in env order.
    kinematics 'holonomic' or 'unicycle': the action space of build_action_space and the robot's propagate; the env's robot
    must step the same kinematics (external_xy / external_rot)."""

    name = 'BatchedValuePolicy'
    trainable = True
    multiagent_training = True

    def __init__(self, model, gamma=0.9, v_pref=1.0, time_step=0.25, joint=True, speed_samples=5, rotation_samples=16,
                 with_om=False, cell_num=4, cell_size=1.0, om_channel_size=3, query_env=True, kinematics='holonomic',
                 order_by_distance=False, exploration='torch', sort_last_state=False):
        if kinematics not in ('holonomic', 'unicycle'):
            raise ValueError('kinematics must be holonomic or unicycle, not %r' % (kinematics,))
        if exploration not in ('torch', 'numpy'):
            raise ValueError('exploration must be torch or numpy, not %r' % (exploration,))
        self.exploration = exploration
        if not joint and not query_env:
            raise ValueError('CADRL always queries the env (cadrl.py:156-170): query_env=False needs a joint policy')
        self.model = model
        self.query_env, self.kinematics, self.order_by_distance = bool(query_env), kinematics, bool(order_by_distance)
        # the rows the reference stores as last_state in the train phase have their humans sorted by decreasing distance
        # to the robot (LSTM-RL: lstm_rl.py:99-104, whatever query_env is); BatchedExplorer records RL pairs in that order
        self.sort_last_state = bool(sort_last_state)
        # policy.config [om] + with_om: occupancy maps of the NEXT human states are appended to every row
        # (multi_human_rl.py:46-49; they do not depend on the action, so they are built once per env and broadcast)
        self.with_om = with_om
        self.om = (cell_num, cell_size, om_channel_size)
        self.gamma = gamma
        self.v_pref, self.time_step = v_pref, time_step
        self.joint = joint
        self.action_space_np = build_action_space(v_pref, speed_samples, rotation_samples, kinematics)
        self.actions = None
        self.device = None
        self.phase = 'test'
        self.epsilon = 0.0                   # train.py:148-152 sets it every episode (policy.set_epsilon)
        self._gen = None; self._seed = 0
        self.action_values = None
        self.explored = None                 # [B] bool: which envs took a random action in the last act_batch (train phase)
        self._buf_states = None; self._buf_reward = None; self._buf_next = None

    def set_device(self, device):
        self.device = torch.device(device)
        self.model.to(self.device)
        self.actions = torch.from_numpy(self.action_space_np).to(self.device)

    def set_phase(self, phase):
        self.phase = phase

    def set_epsilon(self, epsilon):
        """policy.py:37-38"""
        self.epsilon = float(epsilon)

    def set_seed(self, seed):
        """Seed of the exploration draws (per-env uniforms + action indices)."""
        self._seed = int(seed); self._gen = None

    def get_model(self):
        return self.model

    @torch.no_grad()
    def act_batch(self, env):
        if self.actions is None:
            self.set_device(env.device)
        A = self.actions.shape[0]
        B, N = env.B, env.human_num
        # sized per env: one policy may act in envs of different sizes (CADRL trains on one human and tests on N)
        if self._buf_states is None or tuple(self._buf_states.shape[:3]) != (B, A, N):
            self._buf_states = torch.empty((B, A, N, 13), dtype=torch.float32, device=self.device)
            self._buf_reward = torch.empty((B, A), dtype=torch.float64, device=self.device)
        unicycle = self.kinematics == 'unicycle'
        if self.query_env:
            uni = {'unicycle': True} if unicycle else {}              # holonomic: lookahead_pack's default, the call as before
            states, reward = env.lookahead_pack(self.actions, out_states=self._buf_states, out_reward=self._buf_reward, **uni)
        else:
            if self._buf_next is None or tuple(self._buf_next[0].shape[:2]) != (B, N):
                self._buf_next = (torch.empty((B, N, 2), dtype=torch.float64, device=self.device),
                                  torch.empty((B, N, 2), dtype=torch.float64, device=self.device),
                                  torch.empty((B, N), dtype=torch.int32, device=self.device))
            states, reward, npos, nvel, _ = env.propagate_pack(self.actions, unicycle, self.order_by_distance, self._buf_states,
                                                               self._buf_reward, *self._buf_next)
        # multi_human_rl.py:52: pow(gamma, time_step * state.self_state.v_pref) -- the robot's v_pref of THIS env
        discount = torch.pow(torch.full((B,), float(self.gamma), dtype=torch.float64, device=self.device),
                             self.time_step * env.state.r_attr[:, 1]).unsqueeze(1)
        F = 13
        if self.with_om:
            if self.query_env:
                npos, nvel = env.lookahead_humans()
            om = env.occupancy_maps(npos, nvel, *self.om)                # [B][N][cells * channels]
            states = torch.cat([states, om.unsqueeze(1).expand(B, A, N, om.shape[2])], dim=3)
            F = states.shape[3]
        if self.joint:
            v = self.model(states.reshape(B * A, N, F)).view(B, A)
        else:
            v = self.model(states.view(B * A * N, 13)).view(B, A, N).min(dim=2).values
        values = reward + discount * v.double()                        # python-float arithmetic in the reference
        self.action_values = values
        best = values.argmax(dim=1)                                    # the first maximum, like predict's strict >
        self.explored = None
        if self.exploration == 'numpy':                                # every phase draws (multi_human_rl.py:26)
            _, explored, index, reached = env.policy_draws(self.epsilon, A, self.phase == 'train')
            if self.phase == 'train':
                self.explored = explored
                best = torch.where(explored, index, best)
            # the kernel's reach_destination decided which envs drew: the zero action follows the same decision
            act = self.actions[best]
            return torch.where(reached.unsqueeze(1), torch.zeros_like(act), act)
        if self.phase == 'train' and self.epsilon > 0.0:                # epsilon-greedy (multi_human_rl.py:27-31)
            if self._gen is None:
                self._gen = torch.Generator(device=self.device); self._gen.manual_seed(self._seed)
            u = torch.rand((B,), generator=self._gen, device=self.device, dtype=torch.float64)
            rnd = torch.randint(0, A, (B,), generator=self._gen, device=self.device)
            self.explored = u < self.epsilon
            best = torch.where(self.explored, rnd, best)
        act = self.actions[best]
        s = env.state                                                  # policy.py:41-48 reach_destination
        dy, dx = s.r_pos[:, 1] - s.r_goal[:, 1], s.r_pos[:, 0] - s.r_goal[:, 0]
        reached = torch.sqrt(torch.addcmul(dy * dy, dx, dx)) < s.r_attr[:, 0]
        return torch.where(reached.unsqueeze(1), torch.zeros_like(act), act)


def make_sarl(gamma=0.9, v_pref=1.0, time_step=0.25, seed=None, with_om=False, cell_num=4, cell_size=1.0,
              om_channel_size=3, query_env=True, kinematics='holonomic', exploration='torch', speed_samples=5,
              rotation_samples=16, **net_kw):
    """SARL with the reference's default architecture (crowd_nav/configs/policy.config:43-50); random-init weights when
    no checkpoint is loaded (there are no checkpoints in the reference repo). with_om=True gives OM-SARL: input_dim grows
    by cell_num^2 * om_channel_size (multi_human_rl.py:106-107). net_kw: SARLValueNetwork's layer sizes and
    with_global_state."""
    if seed is not None:
        torch.manual_seed(seed)
    if with_om:
        net_kw.setdefault('input_dim', 13 + cell_num * cell_num * om_channel_size)
    p = BatchedValuePolicy(SARLValueNetwork(**net_kw), gamma, v_pref, time_step, joint=True, with_om=with_om,
                           cell_num=cell_num, cell_size=cell_size, om_channel_size=om_channel_size, query_env=query_env,
                           kinematics=kinematics, exploration=exploration, speed_samples=speed_samples,
                           rotation_samples=rotation_samples)
    p.name = 'OM-SARL' if with_om else 'SARL'
    return p


def make_cadrl(gamma=0.9, v_pref=1.0, time_step=0.25, seed=None, kinematics='holonomic', exploration='torch',
               speed_samples=5, rotation_samples=16, mlp_dims=(150, 100, 100, 1)):
    """CADRL queries the env whatever policy.config's query_env says (cadrl.py:156-170), so there is no query_env here."""
    if seed is not None:
        torch.manual_seed(seed)
    p = BatchedValuePolicy(CADRLValueNetwork(mlp_dims=mlp_dims), gamma, v_pref, time_step, joint=False,
                           kinematics=kinematics, exploration=exploration, speed_samples=speed_samples,
                           rotation_samples=rotation_samples)
    p.name = 'CADRL'
    p.multiagent_training = False
    return p


def make_lstm_rl(gamma=0.9, v_pref=1.0, time_step=0.25, seed=None, with_interaction_module=False, query_env=True,
                 kinematics='holonomic', exploration='torch', with_om=False, cell_num=4, cell_size=1.0, om_channel_size=3,
                 speed_samples=5, rotation_samples=16, mlp_dims=(150, 100, 100, 1), lstm_hidden_dim=50,
                 mlp1_dims=(150, 100, 100, 50)):
    """LSTM-RL with the reference's default sizes (crowd_nav/configs/policy.config:24-31). With query_env=False its rows
    follow the reference's sort of the humans by decreasing distance to the robot (lstm_rl.py:99-103); its last_state,
    the rows of its replay pairs, always does (sort_last_state). with_om=True gives OM-LSTM-RL ([lstm_rl] with_om,
    lstm_rl.py:79-88): input_dim grows by cell_num^2 * om_channel_size (multi_human_rl.py:106-107), the LSTM's input or,
    with the interaction module, mlp1's. mlp_dims, lstm_hidden_dim and mlp1_dims are policy.config's [lstm_rl] mlp2_dims,
    global_state_dim and mlp1_dims (lstm_rl.py:77-85)."""
    if seed is not None:
        torch.manual_seed(seed)
    net = LSTMRLValueNetwork(input_dim=13 + (cell_num * cell_num * om_channel_size if with_om else 0),
                             mlp_dims=mlp_dims, lstm_hidden_dim=lstm_hidden_dim,
                             mlp1_dims=mlp1_dims if with_interaction_module else None)
    p = BatchedValuePolicy(net, gamma, v_pref, time_step, joint=True, with_om=with_om, cell_num=cell_num,
                           cell_size=cell_size, om_channel_size=om_channel_size, query_env=query_env, kinematics=kinematics,
                           order_by_distance=not query_env, exploration=exploration, sort_last_state=True,
                           speed_samples=speed_samples, rotation_samples=rotation_samples)
    p.name = 'OM-LSTM-RL' if with_om else 'LSTM-RL'
    return p


def _dims(config, section, key):
    """A layer-size list of policy.config, parsed as the reference parses it (cadrl.py:59)."""
    return [int(x) for x in config.get(section, key).split(', ')]


def _common_parameters(config):
    """CADRL.set_common_parameters (cadrl.py:64-73) as keyword arguments of the make_* builders. [action_space] sampling is
    read and unused, as in the reference (build_action_space always samples speeds exponentially, cadrl.py:82-102)."""
    config.get('action_space', 'sampling')
    return dict(gamma=config.getfloat('rl', 'gamma'), kinematics=config.get('action_space', 'kinematics'),
                speed_samples=config.getint('action_space', 'speed_samples'),
                rotation_samples=config.getint('action_space', 'rotation_samples'),
                query_env=config.getboolean('action_space', 'query_env'), cell_num=config.getint('om', 'cell_num'),
                cell_size=config.getfloat('om', 'cell_size'), om_channel_size=config.getint('om', 'om_channel_size'))


class ConfiguredPolicy(BatchedValuePolicy):
    """A policy_factory entry: built empty, then configure(policy_config) reads the keys the reference's
    policy.configure(config) reads and builds the network and the action space (sarl.py:73-86, lstm_rl.py:75-88,
    cadrl.py:57-72). The configured policy is the one its make_* builder returns for the same values; `exploration`
    ('torch' or 'numpy') is passed on to it."""

    def __init__(self, exploration='torch'):
        self.exploration = exploration
        self.model = None

    def configure(self, config):
        common = _common_parameters(config)
        policy = self.build(config, common)
        self.__dict__.update(policy.__dict__)
        self.speed_samples, self.rotation_samples = common['speed_samples'], common['rotation_samples']

    def build(self, config, common):
        raise NotImplementedError


class CADRL(ConfiguredPolicy):
    """cadrl.py:57-62. CADRL always queries the env, so its query_env is True whatever the config says."""
    name = 'CADRL'

    def build(self, config, common):
        policy = make_cadrl(gamma=common['gamma'], kinematics=common['kinematics'], exploration=self.exploration,
                            speed_samples=common['speed_samples'], rotation_samples=common['rotation_samples'],
                            mlp_dims=_dims(config, 'cadrl', 'mlp_dims'))
        policy.multiagent_training = config.getboolean('cadrl', 'multiagent_training')
        logging.info('Policy: CADRL without occupancy map')
        return policy


class LstmRL(ConfiguredPolicy):
    """lstm_rl.py:75-88: [lstm_rl] mlp2_dims is the value MLP, global_state_dim the LSTM's hidden size, mlp1_dims the
    interaction module's MLP (read only with with_interaction_module). With with_om the name is OM-LSTM-RL, as make_lstm_rl
    names it; the reference keeps 'LSTM-RL' as the attribute and writes 'OM-' only in its log line."""
    name = 'LSTM-RL'

    def build(self, config, common):
        with_interaction_module = config.getboolean('lstm_rl', 'with_interaction_module')
        kw = dict(common, mlp_dims=_dims(config, 'lstm_rl', 'mlp2_dims'),
                  lstm_hidden_dim=config.getint('lstm_rl', 'global_state_dim'),
                  with_om=config.getboolean('lstm_rl', 'with_om'), with_interaction_module=with_interaction_module)
        if with_interaction_module:
            kw['mlp1_dims'] = _dims(config, 'lstm_rl', 'mlp1_dims')
        policy = make_lstm_rl(exploration=self.exploration, **kw)
        policy.multiagent_training = config.getboolean('lstm_rl', 'multiagent_training')
        logging.info('Policy: {}LSTM-RL {} pairwise interaction module'.format(
            'OM-' if kw['with_om'] else '', 'w/' if with_interaction_module else 'w/o'))
        return policy


class SARL(ConfiguredPolicy):
    """sarl.py:73-86"""
    name = 'SARL'

    def build(self, config, common):
        with_om = config.getboolean('sarl', 'with_om')
        with_global_state = config.getboolean('sarl', 'with_global_state')
        kw = dict(common, with_om=with_om, with_global_state=with_global_state,
                  mlp1_dims=_dims(config, 'sarl', 'mlp1_dims'), mlp2_dims=_dims(config, 'sarl', 'mlp2_dims'),
                  mlp3_dims=_dims(config, 'sarl', 'mlp3_dims'), attention_dims=_dims(config, 'sarl', 'attention_dims'))
        policy = make_sarl(exploration=self.exploration, **kw)
        policy.multiagent_training = config.getboolean('sarl', 'multiagent_training')
        logging.info('Policy: {} {} global state'.format(policy.name, 'w/' if with_global_state else 'w/o'))
        return policy


# crowd_nav/policy/policy_factory.py: the trainable policies by the names train.py / test.py take with --policy
policy_factory = {'cadrl': CADRL, 'lstm_rl': LstmRL, 'sarl': SARL}
