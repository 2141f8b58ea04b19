"""python -m crowdnav_b200.train: the reference's crowd_nav/train.py over batched environments on the GPU.

The same flags, output directory, config copies, output.log, checkpoints (il_model.pth, rl_model.pth,
resumed_rl_model.pth) and log lines as train.py:17-173, so the reference's test.py and plot.py read what this writes, with
every rollout streamed through --num_envs environments on device (BatchedExplorer), the replay memory on device
(DeviceReplayMemory) and the SGD steps on the memory's device tensors (trainer.Trainer). New flags:
  --num_envs B                    environments stepped in lockstep (default 1024)
  --exploration numpy|torch       where the epsilon-greedy draws come from: each env's copy of the reference's numpy
                                  stream (default, the reference's exploring actions) or a torch generator
  --yes                           answer the overwrite prompt for an existing output directory with 'y'
--gpu is accepted and changes nothing: the run is always on cuda:0. The reference's git-hash line (train.py:57-58) is not
written.

Imitation learning runs the ORCA robot ([imitation_learning] il_policy = orca; the linear robot is not simulated on
device). A policy with multiagent_training = false (CADRL) trains and validates on one-human circle-crossing scenes, as
the reference's CrowdSim.reset switches to them (crowd_sim.py:265-279): the driver keeps a second env of one human for the
train and val phases and tests on the configured env.
"""
import argparse
import configparser
import logging
import os
import shutil
import sys

import torch


def parse_args(argv=None):
    parser = argparse.ArgumentParser('Parse configuration file')
    parser.add_argument('--env_config', type=str, default='configs/env.config')
    parser.add_argument('--policy', type=str, default='cadrl')
    parser.add_argument('--policy_config', type=str, default='configs/policy.config')
    parser.add_argument('--train_config', type=str, default='configs/train.config')
    parser.add_argument('--output_dir', type=str, default='data/output')
    parser.add_argument('--weights', type=str)
    parser.add_argument('--resume', default=False, action='store_true')
    parser.add_argument('--gpu', default=False, action='store_true')
    parser.add_argument('--debug', default=False, action='store_true')
    parser.add_argument('--num_envs', type=int, default=1024)
    parser.add_argument('--exploration', type=str, default='numpy', choices=['numpy', 'torch'])
    parser.add_argument('--yes', default=False, action='store_true')
    return parser, parser.parse_args(argv)


def read_config(path):
    config = configparser.RawConfigParser()
    if not config.read(path):
        raise FileNotFoundError('cannot read config file %s' % path)
    return config


def setup_logging(log_file, mode, level):
    """train.py:50-56 / test.py:46-47. Replaces the root logger's handlers, so a second run in one process logs to its
    own file."""
    handlers = [logging.StreamHandler(sys.stdout)]
    if log_file is not None:
        handlers.append(logging.FileHandler(log_file, mode=mode))
    logging.basicConfig(level=level, handlers=handlers, format='%(asctime)s, %(levelname)s: %(message)s',
                        datefmt="%Y-%m-%d %H:%M:%S", force=True)


def single_human_config(env_config):
    """The env a policy with multiagent_training = false trains and validates on: one human and circle crossing
    (crowd_sim.py:265-279)."""
    config = configparser.RawConfigParser()
    config.read_dict({section: dict(env_config.items(section)) for section in env_config.sections()})
    config.set('sim', 'human_num', '1')
    config.set('sim', 'train_val_sim', 'circle_crossing')
    return config


def make_env(env_config, num_envs, device):
    from .batched import BatchedCrowdSim
    env = BatchedCrowdSim(num_envs, device)
    env.configure(env_config)
    return env


def fit_policy_to_env(policy, env):
    """What the reference's reset and first predict give a policy (crowd_sim.py:296-298, cadrl.py:146-147): the env's
    time step, and an action space for the robot's v_pref."""
    from .policy import build_action_space
    policy.time_step = env.time_step
    if policy.v_pref != env.robot_v_pref:
        policy.v_pref = env.robot_v_pref
        policy.action_space_np = build_action_space(env.robot_v_pref, policy.speed_samples, policy.rotation_samples,
                                                    policy.kinematics)
        policy.actions = None


def print_info(env, kinematics):
    """agent.py:31-33 for the robot"""
    logging.info('Agent is {} and has {} kinematic constraint'.format(
        'visible' if env.robot_visible else 'invisible', kinematics))


def configure_policy(parser, name, policy_config_file, exploration):
    from .policy import policy_factory
    if name not in policy_factory:
        parser.error('Policy has to be trainable: %s is not one of %s' % (name, ', '.join(sorted(policy_factory))))
    policy = policy_factory[name](exploration=exploration)
    if policy_config_file is None:
        parser.error('Policy config has to be specified for a trainable network')
    policy.configure(read_config(policy_config_file))
    return policy


def main(argv=None, make_env=make_env, explorer_class=None, trainer_class=None, memory_class=None, device=None):
    """train.py:17-173. make_env(env_config, num_envs, device), explorer_class, trainer_class and memory_class build the
    env, BatchedExplorer, Trainer and DeviceReplayMemory; `device` defaults to cuda:0."""
    if explorer_class is None:
        from .explorer import BatchedExplorer as explorer_class
    if trainer_class is None:
        from .trainer import Trainer as trainer_class
    if memory_class is None:
        from .memory import DeviceReplayMemory as memory_class
    parser, args = parse_args(argv)

    # configure paths
    make_new_dir = True
    if os.path.exists(args.output_dir):
        key = 'y' if args.yes else input('Output directory already exists! Overwrite the folder? (y/n)')
        if key == 'y' and not args.resume:
            shutil.rmtree(args.output_dir)
        else:
            make_new_dir = False
            args.env_config = os.path.join(args.output_dir, os.path.basename(args.env_config))
            args.policy_config = os.path.join(args.output_dir, os.path.basename(args.policy_config))
            args.train_config = os.path.join(args.output_dir, os.path.basename(args.train_config))
    if make_new_dir:
        os.makedirs(args.output_dir)
        shutil.copy(args.env_config, args.output_dir)
        shutil.copy(args.policy_config, args.output_dir)
        shutil.copy(args.train_config, args.output_dir)
    log_file = os.path.join(args.output_dir, 'output.log')
    il_weight_file = os.path.join(args.output_dir, 'il_model.pth')
    rl_weight_file = os.path.join(args.output_dir, 'rl_model.pth')

    # configure logging
    setup_logging(log_file, 'a' if args.resume else 'w', logging.INFO if not args.debug else logging.DEBUG)
    device = torch.device('cuda:0') if device is None else torch.device(device)
    logging.info('Using device: %s', device)

    # configure policy
    policy = configure_policy(parser, args.policy, args.policy_config, args.exploration)
    policy.set_device(device)

    # configure environments: the configured one, and one human for the train and val phases of a single-agent policy
    env_config = read_config(args.env_config)
    env = make_env(env_config, args.num_envs, device)
    train_env = env if policy.multiagent_training else make_env(single_human_config(env_config), args.num_envs, device)
    fit_policy_to_env(policy, env)

    # read training parameters
    if args.train_config is None:
        parser.error('Train config has to be specified for a trainable network')
    train_config = read_config(args.train_config)
    rl_learning_rate = train_config.getfloat('train', 'rl_learning_rate')
    train_batches = train_config.getint('train', 'train_batches')
    train_episodes = train_config.getint('train', 'train_episodes')
    sample_episodes = train_config.getint('train', 'sample_episodes')
    target_update_interval = train_config.getint('train', 'target_update_interval')
    evaluation_interval = train_config.getint('train', 'evaluation_interval')
    capacity = train_config.getint('train', 'capacity')
    epsilon_start = train_config.getfloat('train', 'epsilon_start')
    epsilon_end = train_config.getfloat('train', 'epsilon_end')
    epsilon_decay = train_config.getfloat('train', 'epsilon_decay')
    checkpoint_interval = train_config.getint('train', 'checkpoint_interval')

    # configure trainer and explorers: rows of the train env's humans, with the policy's occupancy maps
    feature_dim = 13 + (policy.om[0] ** 2 * policy.om[2] if policy.with_om else 0)
    memory = memory_class(capacity, train_env.human_num, device, feature_dim=feature_dim)
    model = policy.get_model()
    batch_size = train_config.getint('trainer', 'batch_size')
    trainer = trainer_class(model, memory, device, batch_size)
    explorer = explorer_class(train_env, 'orca', device, memory, policy.gamma, target_policy=policy)
    test_explorer = explorer if train_env is env else explorer_class(env, policy, device, gamma=policy.gamma)

    # imitation learning
    if args.resume:
        if not os.path.exists(rl_weight_file):
            logging.error('RL weights does not exist')
        model.load_state_dict(torch.load(rl_weight_file, map_location=device))
        rl_weight_file = os.path.join(args.output_dir, 'resumed_rl_model.pth')
        logging.info('Load reinforcement learning trained weights. Resume training')
    elif os.path.exists(il_weight_file):
        model.load_state_dict(torch.load(il_weight_file, map_location=device))
        logging.info('Load imitation learning trained weights.')
    else:
        il_episodes = train_config.getint('imitation_learning', 'il_episodes')
        il_policy = train_config.get('imitation_learning', 'il_policy')
        il_epochs = train_config.getint('imitation_learning', 'il_epochs')
        il_learning_rate = train_config.getfloat('imitation_learning', 'il_learning_rate')
        if il_policy != 'orca':
            raise ValueError('il_policy = %s is not supported: imitation learning runs the ORCA robot on device '
                             '(set [imitation_learning] il_policy = orca)' % il_policy)
        trainer.set_learning_rate(il_learning_rate)
        if train_env.robot_visible:
            safety_space = 0
        else:
            safety_space = train_config.getfloat('imitation_learning', 'safety_space')
        train_env.robot_safety_space = safety_space
        explorer.run_k_episodes(il_episodes, 'train', update_memory=True, imitation_learning=True)
        trainer.optimize_epoch(il_epochs)
        torch.save(model.state_dict(), il_weight_file)
        logging.info('Finish imitation learning. Weights saved.')
        logging.info('Experience set size: %d/%d', len(memory), memory.capacity)
    explorer.update_target_model(model)

    # reinforcement learning
    explorer.robot_policy = policy
    print_info(env, policy.kinematics)
    trainer.set_learning_rate(rl_learning_rate)
    # fill the memory pool with some RL experience
    if args.resume:
        policy.set_epsilon(epsilon_end)
        policy.set_phase('train')
        explorer.run_k_episodes(100, 'train', update_memory=True, episode=0)
        logging.info('Experience set size: %d/%d', len(memory), memory.capacity)
    episode = 0
    while episode < train_episodes:
        if args.resume:
            epsilon = epsilon_end
        else:
            if episode < epsilon_decay:
                epsilon = epsilon_start + (epsilon_end - epsilon_start) / epsilon_decay * episode
            else:
                epsilon = epsilon_end
        policy.set_epsilon(epsilon)

        # evaluate the model
        if episode % evaluation_interval == 0:
            policy.set_phase('val')
            explorer.run_k_episodes(train_env.case_size['val'], 'val', episode=episode)

        # sample k episodes into memory and optimize over the generated memory
        policy.set_phase('train')
        explorer.run_k_episodes(sample_episodes, 'train', update_memory=True, episode=episode)
        trainer.optimize_batch(train_batches)
        episode += 1

        if episode % target_update_interval == 0:
            explorer.update_target_model(model)

        if episode != 0 and episode % checkpoint_interval == 0:
            torch.save(model.state_dict(), rl_weight_file)

    # final test
    policy.set_phase('test')
    test_explorer.run_k_episodes(env.case_size['test'], 'test', episode=episode)


if __name__ == '__main__':
    main()
