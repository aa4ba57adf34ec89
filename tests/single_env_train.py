"""The single-environment training loop that train.train ran before it learned to step several environments (reference
train.py:23-216 over the replay environment), kept verbatim as the yardstick for ``train.train(num_envs=1)``: the same
calls, noise draws, permutations and weights.  ``PPO`` and the other collaborators are looked up in this module's globals,
so a CPU test can substitute recording fakes."""
import os
import random
import shutil

import numpy as np

from carla_ppo_b200.ppo import PPO
from carla_ppo_b200.replay_env import ReplayEnv, reward_functions
from carla_ppo_b200.run_eval import run_eval
from carla_ppo_b200.train import load_replay_frames
from carla_ppo_b200.utils import compute_gae
from carla_ppo_b200.vae_common import create_encode_state_fn, load_vae


def train_one_env(params, start_carla=False, restart=False, env=None, vae=None, models_root="models", interactive=True):
    """train.train as it was before --num_envs, verbatim: one environment, one episode per update block."""
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
    if env is None:
        print("Creating environment")
        env = ReplayEnv(load_replay_frames(params.get("replay_data", "vae/data")), obs_res=(160, 80),
                        action_smoothing=params["action_smoothing"], encode_state_fn=None,
                        reward_fn=reward_functions[params["reward_fn"]], synchronous=params["synchronous"], fps=params["fps"],
                        start_carla=False, episode_length=params.get("episode_length", 256))
    if isinstance(seed, int):
        env.seed(seed)
    best_eval_reward = -float("inf")

    input_shape = np.array([vae.z_dim + len(measurements_to_include)])
    print("Creating model")
    model = PPO(input_shape, env.action_space, learning_rate=learning_rate, lr_decay=lr_decay, epsilon=ppo_epsilon,
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

    actor = None
    if fused:
        from carla_ppo_b200.actor import FusedActor
        actor = FusedActor(vae, model, measurements_to_include)
        env.encode_state_fn = actor.encode_state_fn
        predict = actor.predict
    else:
        env.encode_state_fn = create_encode_state_fn(vae, measurements_to_include)
        predict = model.predict

    def log_episode(prefix, episode_idx):
        model.write_value_to_summary(prefix + "/distance_traveled", env.distance_traveled, episode_idx)
        model.write_value_to_summary(prefix + "/average_speed", 3.6 * env.speed_accum / max(env.step_count, 1), episode_idx)
        model.write_value_to_summary(prefix + "/center_lane_deviation", env.center_lane_deviation, episode_idx)
        model.write_value_to_summary(prefix + "/average_center_lane_deviation", env.center_lane_deviation / max(env.step_count, 1), episode_idx)
        model.write_value_to_summary(prefix + "/distance_over_deviation", env.distance_traveled / max(env.center_lane_deviation, 1e-9), episode_idx)

    history = []
    while num_episodes <= 0 or model.get_episode_idx() < num_episodes:
        episode_idx = model.get_episode_idx()
        if episode_idx % eval_interval == 0:
            video_filename = os.path.join(model.video_dir, "episode{}.avi".format(episode_idx)) if params.get("record_eval") else None
            eval_reward = run_eval(env, model, video_filename=video_filename, actor=actor)
            model.write_value_to_summary("eval/reward", eval_reward, episode_idx)
            log_episode("eval", episode_idx)
            if eval_reward > best_eval_reward:
                model.save()
                best_eval_reward = eval_reward

        state, terminal_state, total_reward = env.reset(), False, 0
        print(f"Episode {episode_idx} (Step {model.get_train_step_idx()})")
        while not terminal_state:
            states, taken_actions, values, rewards, dones = [], [], [], [], []
            for _ in range(horizon):
                action, value = predict(state, write_to_summary=True)
                new_state, reward, terminal_state, info = env.step(action)
                if info["closed"]:
                    return model
                env.extra_info.extend(["Episode {}".format(episode_idx), "Training...", "", "Value:  % 20.2f" % value])
                env.render()
                total_reward += reward
                states.append(state); taken_actions.append(action); values.append(value)
                rewards.append(reward); dones.append(terminal_state)
                state = new_state
                if terminal_state:
                    break
            _, last_values = predict(state)                              # bootstrap value (train.py:172)
            T = len(rewards)
            if reference_loop:
                advantages = compute_gae(rewards, values, last_values, dones, discount_factor, gae_lambda)
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
                model.learn(np.array(states), np.array(taken_actions), values, rewards, dones, last_values, gamma=discount_factor,
                            lam=gae_lambda, num_epochs=num_epochs, batch_size=batch_size, perms=np.stack(perms) if perms else None)
        model.write_value_to_summary("train/reward", total_reward, episode_idx)
        log_episode("train", episode_idx)
        model.write_episodic_summaries()
        history.append(total_reward)
    model.reward_history = history
    return model
