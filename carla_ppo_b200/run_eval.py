"""Drop-in for the reference's ``run_eval.py``: ``run_eval(env, model, video_filename=None)`` (run_eval.py:30-73) and the
CLI (:75-141) over the offline replay environment.  ``model`` is anything with ``predict(state, greedy=True)`` and
``get_episode_idx()`` -- the PPO class or a FusedActor-backed one."""
from __future__ import annotations

import os

import numpy as np


def run_eval(env, model, video_filename=None, actor=None):
    """One greedy episode (std = 0, run_eval.py:51); returns the total reward.  ``actor`` (FusedActor, optional) serves
    the per-step encode + predict in one C call."""
    if actor is not None:
        actor.greedy = True
    try:
        state, terminal, total_reward = env.reset(is_training=False), False, 0
        rendered_frame = env.render(mode="rgb_array")
        recorder = None
        if video_filename is not None and rendered_frame is not None:
            from .utils import VideoRecorder
            print("Recording video to {} ({}x{}x{}@{}fps)".format(video_filename, *rendered_frame.shape, int(env.average_fps)))
            recorder = VideoRecorder(video_filename, frame_size=rendered_frame.shape, fps=env.average_fps)
            recorder.add_frame(rendered_frame)
        episode_idx = model.get_episode_idx()
        info = {"closed": False}
        predict = actor.predict if actor is not None else model.predict
        while not terminal:
            env.extra_info.append("Episode {}".format(episode_idx))
            env.extra_info.append("Running eval...")
            env.extra_info.append("")
            action, _ = predict(state, greedy=True)                  # deterministic actions at test time
            state, reward, terminal, info = env.step(action)
            if info["closed"]:
                break
            rendered_frame = env.render(mode="rgb_array")
            if recorder is not None:
                recorder.add_frame(rendered_frame)
            total_reward += reward
        if recorder is not None:
            recorder.release()
        return total_reward
    finally:
        if actor is not None:
            actor.greedy = False


def main(argv=None):
    import argparse
    from .actor import FusedActor
    from .ppo import PPO
    from .replay_env import ReplayEnv, reward_functions
    from .train import load_replay_frames
    from .vae_common import create_encode_state_fn, load_vae
    parser = argparse.ArgumentParser(description="Runs the model in evaluation mode (offline replay environment)")
    parser.add_argument("--model_name", type=str, required=True)
    parser.add_argument("--reward_fn", type=str, default="reward_speed_centering_angle_multiply")
    parser.add_argument("--vae_model", type=str, default="vae/models/seg_bce_cnn_zdim64_beta1_kl_tolerance0.0_data/")
    parser.add_argument("--vae_model_type", type=str, default=None)
    parser.add_argument("--vae_z_dim", type=int, default=None)
    parser.add_argument("--synchronous", type=int, default=True)
    parser.add_argument("--fps", type=int, default=30)
    parser.add_argument("--action_smoothing", type=float, default=0.0)
    parser.add_argument("-start_carla", action="store_true", help="accepted and ignored: there is no simulator to start")
    parser.add_argument("--record_to_file", type=str, default=None)
    parser.add_argument("--replay_data", type=str, default="vae/data", help="directory with rgb/*.png (or a .npz with 'rgb') to replay")
    parser.add_argument("--models_root", type=str, default="models")
    parser.add_argument("--unfused", action="store_true", help="separate encode / predict calls like the reference")
    args = parser.parse_args(argv)

    vae = load_vae(args.vae_model, args.vae_z_dim, args.vae_model_type)
    measurements_to_include = set(["steer", "throttle", "speed"])
    obs_res = (vae.source_shape[1], vae.source_shape[0])                  # (width, height) of the frames the VAE takes
    env = ReplayEnv(load_replay_frames(args.replay_data), obs_res=obs_res, action_smoothing=args.action_smoothing,
                    encode_state_fn=create_encode_state_fn(vae, measurements_to_include), reward_fn=reward_functions[args.reward_fn],
                    synchronous=args.synchronous, fps=args.fps, start_carla=False)
    np.random.seed(0)
    env.seed(0)
    input_shape = np.array([vae.z_dim + len(measurements_to_include)])
    model = PPO(input_shape, env.action_space, model_dir=os.path.join(args.models_root, args.model_name), seed=0)
    model.init_session(init_logging=False)
    model.load_latest_checkpoint()
    actor = None
    if not args.unfused:
        actor = FusedActor(vae, model, measurements_to_include)
        env.encode_state_fn = actor.encode_state_fn
    print("Running eval...")
    total = run_eval(env, model, video_filename=args.record_to_file, actor=actor)
    print("Done! total reward %.3f" % total)
    env.close()
    return total


if __name__ == "__main__":
    main()
