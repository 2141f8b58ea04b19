"""python -m crowdnav_b200.test: the reference's crowd_nav/test.py over batched environments on the GPU.

The same flags and weight-file choice (test.py:31-43: il_model.pth with --il, else resumed_rl_model.pth when it exists,
else rl_model.pth), --square / --circle, ORCA's safety space and the run of run_k_episodes(case_size[phase], phase,
print_failure=True), with every case streamed through --num_envs environments on device (BatchedExplorer) and the same
log lines. --policy is orca (the robot's ORCA runs inside the step kernels) or one of the trainable policies of
policy.policy_factory. --human_times adds the humans' average time to goal over the successful cases
(BatchedExplorer(human_times=True)). Rendering (--visualize, --traj, --video_file) is not provided. --gpu is accepted and
changes nothing: the run is always on cuda:0.
"""
import argparse
import logging
import os

import torch

from .train import fit_policy_to_env, make_env, print_info, read_config, setup_logging


def parse_args(argv=None):
    parser = argparse.ArgumentParser('Parse configuration file')
    parser.add_argument('--env_config', type=str, default='configs/env.config')
    parser.add_argument('--policy_config', type=str, default='configs/policy.config')
    parser.add_argument('--policy', type=str, default='orca')
    parser.add_argument('--model_dir', type=str, default=None)
    parser.add_argument('--il', default=False, action='store_true')
    parser.add_argument('--gpu', default=False, action='store_true')
    parser.add_argument('--visualize', default=False, action='store_true')
    parser.add_argument('--phase', type=str, default='test')
    parser.add_argument('--test_case', type=int, default=None)
    parser.add_argument('--square', default=False, action='store_true')
    parser.add_argument('--circle', default=False, action='store_true')
    parser.add_argument('--video_file', type=str, default=None)
    parser.add_argument('--traj', default=False, action='store_true')
    parser.add_argument('--num_envs', type=int, default=1024)
    parser.add_argument('--human_times', default=False, action='store_true')
    return parser, parser.parse_args(argv)


def weight_file(model_dir, il):
    """test.py:34-40"""
    if il:
        return os.path.join(model_dir, 'il_model.pth')
    if os.path.exists(os.path.join(model_dir, 'resumed_rl_model.pth')):
        return os.path.join(model_dir, 'resumed_rl_model.pth')
    return os.path.join(model_dir, 'rl_model.pth')


def main(argv=None, make_env=make_env, explorer_class=None, device=None):
    """test.py:14-109 without rendering; returns run_k_episodes' statistics."""
    if explorer_class is None:
        from .explorer import BatchedExplorer as explorer_class
    from .policy import policy_factory
    parser, args = parse_args(argv)
    if args.visualize or args.traj or args.video_file is not None:
        parser.error('rendering (--visualize, --traj, --video_file) is not provided by the batched test driver; '
                     'run the reference\'s test.py for a single rendered case')
    if args.policy != 'orca' and args.policy not in policy_factory:
        parser.error('unknown policy %s: orca or one of %s' % (args.policy, ', '.join(sorted(policy_factory))))

    if args.model_dir is not None:
        env_config_file = os.path.join(args.model_dir, os.path.basename(args.env_config))
        policy_config_file = os.path.join(args.model_dir, os.path.basename(args.policy_config))
        model_weights = weight_file(args.model_dir, args.il)
    else:
        env_config_file = args.env_config
        policy_config_file = args.policy_config

    # configure logging and device
    setup_logging(None, None, logging.INFO)
    device = torch.device('cuda:0') if device is None else torch.device(device)
    logging.info('Using device: %s', device)

    # configure policy
    if args.policy == 'orca':
        policy = 'orca'
    else:
        if args.model_dir is None:
            parser.error('Trainable policy must be specified with a model weights directory')
        policy = policy_factory[args.policy]()
        policy.configure(read_config(policy_config_file))
        policy.get_model().load_state_dict(torch.load(model_weights, map_location=device))

    # configure environment
    env = make_env(read_config(env_config_file), args.num_envs, device)
    if args.square:
        env.test_sim = 'square_crossing'
    if args.circle:
        env.test_sim = 'circle_crossing'
    explorer = explorer_class(env, policy, device, gamma=0.9, human_times=args.human_times)

    if policy == 'orca':
        # test.py:77-85: no safety space for ORCA, visible robot or not
        env.robot_safety_space = 0
        logging.info('ORCA agent buffer: %f', env.robot_safety_space)
        print_info(env, 'holonomic')
    else:
        policy.set_phase(args.phase)
        policy.set_device(device)
        fit_policy_to_env(policy, env)
        print_info(env, policy.kinematics)
    return explorer.run_k_episodes(env.case_size[args.phase], args.phase, print_failure=True)


if __name__ == '__main__':
    main()
