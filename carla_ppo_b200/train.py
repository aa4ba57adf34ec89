"""Drop-in for the reference's ``train.py`` (train.py:23-216 ``train(params, start_carla, restart)`` and the CLI :218-276) over
the offline replay environment (SURVEY.md section 8f-3): the same episode / horizon / update structure, the same
hyper-parameter flags and TensorBoard tags, with the neural work on the H100 library:

  * every environment step:  FusedActor = VAE encode + PPO predict in one C call (cpb_encode_predict) instead of two
    TensorFlow session runs                                                              (train.py:143 + vae_common.py:45-61)
  * every update:            PPO.learn = GAE, returns, advantage normalisation, theta_old <- theta and the
                             num_epochs x ceil(T/batch) minibatch Adam steps in one C call (train.py:171-207);
                             ``--reference_loop`` runs the reference's own Python loop over PPO.train instead
                             (numerically identical: tests/test_integration_gpu.py)
  * ``--num_envs N``:        N replay environments (seeded seed + i) in lockstep: one batched encode + predict per step
                             (B = number of active environments) and one update per rollout over one trajectory segment
                             per environment (PPO.learn(segment_lengths=...)); N = 1 is the reference's loop
"""
from __future__ import annotations

import os
import random
import shutil

import numpy as np

from .ppo import PPO
from .replay_env import ReplayEnv, reward_functions
from .run_eval import run_eval
from .utils import compute_gae
from .vae_common import create_encode_state_fn, load_vae


def load_replay_frames(path, limit=None):
    """uint8 [N,H,W,3] frames from a directory laid out like the reference's vae/data (rgb/{i}.png), a .npz with an
    'rgb' array (tests/golden/frames_u8.npz), or an array."""
    if not isinstance(path, str):
        return np.asarray(path)
    if os.path.isfile(path) and path.endswith(".npz"):
        return np.load(path)["rgb"][:limit]
    from PIL import Image
    d = os.path.join(path, "rgb") if os.path.isdir(os.path.join(path, "rgb")) else path
    names = sorted((f for f in os.listdir(d) if f.endswith(".png")), key=lambda f: int(os.path.splitext(f)[0]) if os.path.splitext(f)[0].isdigit() else 0)
    names = names[:limit] if limit else names
    if not names:
        raise FileNotFoundError("no PNG frames under %s" % d)
    return np.stack([np.asarray(Image.open(os.path.join(d, f)))[:, :, :3] for f in names])


def train(params, start_carla=False, restart=False, env=None, vae=None, models_root="models", interactive=True):
    """reference train.py:23-216.  ``env`` / ``vae`` may be passed in (tests); otherwise a ReplayEnv over
    ``params["replay_data"]`` and ``load_vae(params["vae_model"], ...)`` are created.  Returns the PPO model."""
    learning_rate = params["learning_rate"]; lr_decay = params["lr_decay"]
    discount_factor = params["discount_factor"]; gae_lambda = params["gae_lambda"]
    ppo_epsilon = params["ppo_epsilon"]; initial_std = params["initial_std"]
    value_scale = params["value_scale"]; entropy_scale = params["entropy_scale"]
    horizon = params["horizon"]; num_epochs = params["num_epochs"]
    num_episodes = params["num_episodes"]; batch_size = params["batch_size"]
    model_name = params["model_name"]; seed = params["seed"]
    eval_interval = params["eval_interval"]
    fused = not params.get("unfused", False)
    reference_loop = params.get("reference_loop", False)

    if isinstance(seed, int):
        np.random.seed(seed)
        random.seed(0)

    if vae is None:
        vae = load_vae(params["vae_model"], params["vae_z_dim"], params["vae_model_type"])
    params["vae_z_dim"] = vae.z_dim
    params["vae_model_type"] = "mlp" if type(vae).__name__ == "MlpVAE" else "cnn"
    print("")
    print("Training parameters:")
    for k, v in params.items():
        print(f"  {k}: {v}")
    print("")

    measurements_to_include = set(["steer", "throttle", "speed"])
    num_envs = int(params.get("num_envs", 1))
    if num_envs < 1:
        raise ValueError("num_envs must be >= 1")
    if env is None:
        print("Creating environment")
        frames = load_replay_frames(params.get("replay_data", "vae/data"))
        obs_res = (vae.source_shape[1], vae.source_shape[0])          # (width, height) of the frames the VAE takes
        envs = [ReplayEnv(frames, obs_res=obs_res, action_smoothing=params["action_smoothing"], encode_state_fn=None,
                          reward_fn=reward_functions[params["reward_fn"]], synchronous=params["synchronous"], fps=params["fps"],
                          start_carla=False, episode_length=params.get("episode_length", 256)) for _ in range(num_envs)]
    else:
        envs = list(env) if isinstance(env, (list, tuple)) else [env]
        if len(envs) != num_envs:
            raise ValueError("num_envs = %d but %d environments were given" % (num_envs, len(envs)))
    if isinstance(seed, int):
        for i, e in enumerate(envs):
            e.seed(seed + i)
    best_eval_reward = -float("inf")

    input_shape = np.array([vae.z_dim + len(measurements_to_include)])
    print("Creating model")
    model = PPO(input_shape, envs[0].action_space, learning_rate=learning_rate, lr_decay=lr_decay, epsilon=ppo_epsilon,
                initial_std=initial_std, value_scale=value_scale, entropy_scale=entropy_scale,
                model_dir=os.path.join(models_root, model_name), seed=seed if isinstance(seed, int) else None)
    if not restart and interactive:
        if os.path.isdir(model.log_dir) and len(os.listdir(model.log_dir)) > 0:
            answer = input("Model \"{}\" already exists. Do you wish to continue (C) or restart training (R)? ".format(model_name))
            if answer.upper() == "R":
                restart = True
            elif answer.upper() != "C":
                raise Exception("There are already log files for model \"{}\". Please delete it or change model_name and try again".format(model_name))
    if restart:
        shutil.rmtree(model.model_dir)
        for d in model.dirs:
            os.makedirs(d)
    model.init_session(init_logging=params.get("logging", True))
    if not restart:
        model.load_latest_checkpoint()
    model.write_dict_to_summary("hyperparameters", params, 0)

    # Training steps every environment, then encodes all of their new frames and predicts their actions in one batched
    # call (actor.encode_predict); the environments' own encode_state_fn does nothing meanwhile.  Evaluation runs the
    # single-environment callback on envs[0].
    actor = None
    if fused:
        from .actor import FusedActor
        actor = FusedActor(vae, model, measurements_to_include)
        vec_actor, eval_encode_state_fn = actor, actor.encode_state_fn
    else:
        from .actor import UnfusedActor
        vec_actor, eval_encode_state_fn = UnfusedActor(vae, model, measurements_to_include), create_encode_state_fn(vae, measurements_to_include)
    for e in envs:
        e.encode_state_fn = _deferred_encode

    def log_episode(prefix, episode_idx, logged):
        mean = lambda f: float(np.mean([f(e) for e in logged]))
        model.write_value_to_summary(prefix + "/distance_traveled", mean(lambda e: e.distance_traveled), episode_idx)
        model.write_value_to_summary(prefix + "/average_speed", mean(lambda e: 3.6 * e.speed_accum / max(e.step_count, 1)), episode_idx)
        model.write_value_to_summary(prefix + "/center_lane_deviation", mean(lambda e: e.center_lane_deviation), episode_idx)
        model.write_value_to_summary(prefix + "/average_center_lane_deviation", mean(lambda e: e.center_lane_deviation / max(e.step_count, 1)), episode_idx)
        model.write_value_to_summary(prefix + "/distance_over_deviation", mean(lambda e: e.distance_traveled / max(e.center_lane_deviation, 1e-9)), episode_idx)

    def log_sampled_actions(actions):
        """What predict(state, write_to_summary=True) records for each action taken (ppo.py:248)."""
        for act in actions:
            if model.train_writer is not None:
                for k in range(model.num_actions):
                    model.train_writer.add_scalar("predict_actor/action_%d/sampled_action" % k, float(act[k]), model.predict_step_counter)
            model.predict_step_counter += 1

    history = []
    # One round = every environment plays one training episode (the reference's episode at num_envs = 1).  A rollout
    # steps the still-active environments in lockstep for up to `horizon` steps; an environment that terminates stops
    # collecting for the rest of the round (the reference's `break`).  Each rollout ends in ONE update over one trajectory
    # segment per environment that collected rows, in environment order.
    while num_episodes <= 0 or model.get_episode_idx() < num_episodes:
        episode_idx = model.get_episode_idx()
        if episode_idx % eval_interval == 0:
            video_filename = os.path.join(model.video_dir, "episode{}.avi".format(episode_idx)) if params.get("record_eval") else None
            envs[0].encode_state_fn = eval_encode_state_fn
            eval_reward = run_eval(envs[0], model, video_filename=video_filename, actor=actor)
            envs[0].encode_state_fn = _deferred_encode
            model.write_value_to_summary("eval/reward", eval_reward, episode_idx)
            log_episode("eval", episode_idx, envs[:1])
            if eval_reward > best_eval_reward:
                model.save()
                best_eval_reward = eval_reward

        for e in envs:
            e.reset()
        # state / action / value of every environment: the prediction for its current state
        state, action, value = (list(x) for x in vec_actor.encode_predict(envs))
        total_reward = [0.0] * num_envs
        active = list(range(num_envs))
        print(f"Episode {episode_idx} (Step {model.get_train_step_idx()})")
        first_rollout = True
        while active:
            if not first_rollout:                     # the reference predicts again on the state it bootstrapped from
                a, v = model.predict(np.stack([state[i] for i in active]))
                a, v = np.reshape(a, (len(active), -1)), np.reshape(v, (len(active),))
                for j, i in enumerate(active):
                    action[i], value[i] = a[j], v[j]
            first_rollout = False
            rollout = {i: ([], [], [], [], []) for i in active}      # states, taken_actions, values, rewards, dones
            for _ in range(horizon):
                log_sampled_actions([action[i] for i in active])
                stepped, terminal = list(active), {}
                for i in stepped:
                    _, reward, terminal[i], info = envs[i].step(action[i])
                    if info["closed"]:
                        return model
                    envs[i].extra_info.extend(["Episode {}".format(episode_idx), "Training...", "", "Value:  % 20.2f" % value[i]])
                    envs[i].render()
                    total_reward[i] += reward
                    for buf, x in zip(rollout[i], (state[i], action[i], value[i], reward, terminal[i])):
                        buf.append(x)
                new_state, new_action, new_value = vec_actor.encode_predict([envs[i] for i in stepped])
                for j, i in enumerate(stepped):
                    state[i], action[i], value[i] = new_state[j], new_action[j], new_value[j]
                active = [i for i in stepped if not terminal[i]]
                if not active:
                    break
            # bootstrap values (train.py:172): the predictions on each environment's current state
            segments = [i for i in sorted(rollout) if rollout[i][3]]
            states, taken_actions, values, rewards, dones = ([x for i in segments for x in rollout[i][k]] for k in range(5))
            last_values = [value[i] for i in segments]
            lengths = [len(rollout[i][3]) for i in segments]
            T = len(rewards)
            if reference_loop:
                advantages = np.concatenate([compute_gae(rollout[i][3], rollout[i][2], value[i], rollout[i][4], discount_factor, gae_lambda)
                                             for i in segments])
                returns = advantages + values
                advantages = (advantages - advantages.mean()) / (advantages.std() + 1e-8)
                s_arr, a_arr = np.array(states), np.array(taken_actions)
                model.update_old_policy()
                for _ in range(num_epochs):
                    indices = np.arange(T)
                    np.random.shuffle(indices)
                    for i in range(int(np.ceil(T / batch_size))):
                        mb_idx = indices[i * batch_size:(i + 1) * batch_size]
                        model.train(s_arr[mb_idx], a_arr[mb_idx], returns[mb_idx], advantages[mb_idx])
            else:
                perms = []
                for _ in range(num_epochs):                               # the same np.random.shuffle stream as the loop above
                    indices = np.arange(T)
                    np.random.shuffle(indices)
                    perms.append(indices)
                if num_envs == 1:
                    model.learn(np.array(states), np.array(taken_actions), values, rewards, dones, last_values[0],
                                gamma=discount_factor, lam=gae_lambda, num_epochs=num_epochs, batch_size=batch_size,
                                perms=np.stack(perms) if perms else None)
                else:
                    model.learn(np.array(states), np.array(taken_actions), values, rewards, dones, last_values,
                                gamma=discount_factor, lam=gae_lambda, num_epochs=num_epochs, batch_size=batch_size,
                                perms=np.stack(perms) if perms else None, segment_lengths=lengths)
        model.write_value_to_summary("train/reward", float(np.mean(total_reward)), episode_idx)
        log_episode("train", episode_idx, envs)
        model.write_episodic_summaries()
        history.append(float(np.mean(total_reward)))
    model.reward_history = history
    return model


def _deferred_encode(env):
    """encode_state_fn of the training environments: the loop encodes all stepped environments in one call afterwards."""
    return None


def main(argv=None):
    import argparse
    parser = argparse.ArgumentParser(description="Trains an agent with PPO on the offline replay environment")
    parser.add_argument("--learning_rate", type=float, default=1e-4)
    parser.add_argument("--lr_decay", type=float, default=1.0)
    parser.add_argument("--discount_factor", type=float, default=0.99)
    parser.add_argument("--gae_lambda", type=float, default=0.95)
    parser.add_argument("--ppo_epsilon", type=float, default=0.2)
    parser.add_argument("--initial_std", type=float, default=1.0)
    parser.add_argument("--value_scale", type=float, default=1.0)
    parser.add_argument("--entropy_scale", type=float, default=0.01)
    parser.add_argument("--horizon", type=int, default=128)
    parser.add_argument("--num_epochs", type=int, default=3)
    parser.add_argument("--batch_size", type=int, default=32)
    parser.add_argument("--num_episodes", type=int, default=0)
    parser.add_argument("--vae_model", type=str, default="vae/models/seg_bce_cnn_zdim64_beta1_kl_tolerance0.0_data/")
    parser.add_argument("--vae_model_type", type=str, default=None)
    parser.add_argument("--vae_z_dim", type=int, default=None)
    parser.add_argument("--synchronous", type=int, default=True)
    parser.add_argument("--fps", type=int, default=30)
    parser.add_argument("--action_smoothing", type=float, default=0.0)
    parser.add_argument("-start_carla", action="store_true", help="accepted and ignored: there is no simulator to start")
    parser.add_argument("--model_name", type=str, required=True)
    parser.add_argument("--reward_fn", type=str, default="reward_speed_centering_angle_multiply")
    parser.add_argument("--seed", type=int, default=0)
    parser.add_argument("--eval_interval", type=int, default=5)
    parser.add_argument("--record_eval", type=bool, default=False)
    parser.add_argument("-restart", action="store_true")
    # additions of this build
    parser.add_argument("--replay_data", type=str, default="vae/data", help="recorded frames to replay (dir with rgb/*.png, or .npz)")
    parser.add_argument("--episode_length", type=int, default=256)
    parser.add_argument("--models_root", type=str, default="models")
    parser.add_argument("--unfused", action="store_true", help="separate encode / predict calls per step, like the reference")
    parser.add_argument("--reference_loop", action="store_true", help="the reference's Python minibatch loop over PPO.train instead of PPO.learn")
    parser.add_argument("--num_envs", type=int, default=1, help="replay environments stepped in lockstep (seeded seed + i); "
                        "one batched encode + predict per step and one PPO update over all their rollouts")
    params = vars(parser.parse_args(argv))
    start_carla = params.pop("start_carla")
    restart = params.pop("restart")
    models_root = params.pop("models_root")
    return train(params, start_carla, restart, models_root=models_root)


if __name__ == "__main__":
    main()
