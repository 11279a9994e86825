"""GPU: a whole `update_params` iteration (values -> GAE -> fixed log-probs -> epochs x minibatches, reference
urban_planning_agent.py:248-361) on the H100 path against the padded eager-PyTorch oracle port driven by the same
np.random permutations; and the drop-in nn.Modules dispatching to the CUDA library."""
import math

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from harness import Agent, Cfg, rel, tensorfy
from oracle import torch_port as TP

pytestmark = pytest.mark.gpu


def port_update_params(flat, states, actions, rewards, masks, exps, gamma, tau, epochs, B, seed):
    """The reference's update_params/update_policy control flow on the oracle port (CPU)."""
    agent = TP.PortAgent(flat)
    T = len(states)
    b_all = TP.stack_states(states)
    act = torch.tensor(actions)
    with torch.no_grad():
        values = TP.value(agent.params(), b_all)
    adv, ret = TP.estimate_advantages(torch.tensor(rewards), torch.tensor(masks), values, gamma, tau)
    with torch.no_grad():
        fixed, _ = TP.log_prob_entropy(agent.params(), b_all, act)
    exps_t = torch.tensor(exps)
    np.random.seed(seed)
    losses = []
    order = np.arange(T)
    for _ in range(epochs):
        perm = np.arange(T)
        np.random.shuffle(perm)
        order = order[perm]          # the reference permutes the already permuted lists (urban_planning_agent.py:306-312)
        for i in range(int(math.floor(T / B))):
            idx = order[i * B:(i + 1) * B]
            b = TP.stack_states([states[j] for j in idx])
            ind = exps_t[idx].nonzero(as_tuple=False).squeeze(1)
            losses.append(agent.step(b, act[idx], adv[idx], ret[idx], fixed[idx], ind))
    return agent.flat(), np.array(losses), adv.numpy(), ret.numpy(), fixed.numpy()


def test_update_params_iteration_matches_oracle_port():
    from drl_urban_planning_b200.ppo import PPOUpdater
    dev = torch.device("cuda", 0)
    T, B, epochs = 72, 16, 2
    states, actions = synth.make_states(41, "small", T)
    rng = np.random.default_rng(41)
    rewards = rng.standard_normal(T).astype(np.float32)
    masks = np.ones(T, np.float32); masks[11::12] = 0.0
    exps = np.ones(T, np.float32); exps[5] = 0.0
    flat = PL.default_init(41)
    want, want_losses, adv, ret, fixed = port_update_params(flat, states, actions, rewards, masks, exps, 0.99, 0.95,
                                                           epochs, B, seed=7)
    spec = synth.COMMUNITIES["small"]
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, gamma=0.99, tau=0.95, opt_num_epochs=epochs,
                    mini_batch_size=B, clip_mode=_lib.CLIP_REFERENCE)
    logged = []
    np.random.seed(7)
    up.update_params(states, actions, rewards, masks, exps, log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    assert rel(up.advantages.cpu().numpy(), adv.ravel()) < 1e-5
    assert rel(up.fixed_log_probs.cpu().numpy(), fixed.ravel()) < 1e-5
    got_losses = np.array([v for tag, v, s in logged if tag == "loss/loss"])
    assert got_losses.shape[0] == epochs * (T // B)
    assert np.allclose(got_losses, want_losses[:, 0], rtol=2e-4, atol=2e-5)
    assert rel(up.flat_params(), want) < 2e-5
    steps = [s for tag, v, s in logged if tag == "loss/value_loss"]
    assert steps == list(range(epochs * (T // B)))          # same TensorBoard step indices as the reference


def test_update_params_matches_reference_update_policy(golden_dir):
    """The whole iteration against the trajectory of the UNMODIFIED reference's update_params / update_policy
    (tests/golden/make_golden.py::run_update_params): 3 epochs, so the composition of the epoch permutations
    (urban_planning_agent.py:306-312) matters from epoch 2 on; per-minibatch losses, TensorBoard totals and the final
    parameters."""
    import os
    from drl_urban_planning_b200.ppo import PPOUpdater
    from fixtures_io import expand_states
    z = np.load(os.path.join(golden_dir, "update_small.npz"))
    T, B, epochs, np_seed = (int(x) for x in z["cfg"])
    states = expand_states(z)
    dev = torch.device("cuda", 0)
    up = PPOUpdater(z["params"], int(z["n_cap"]), int(z["e_cap"]), dev, gamma=float(z["gamma_tau"][0]),
                    tau=float(z["gamma_tau"][1]), opt_num_epochs=epochs, mini_batch_size=B,
                    clip_mode=_lib.CLIP_REFERENCE)
    logged = []
    np.random.seed(np_seed)
    out = up.update_params(states, z["actions"], z["rewards"], z["masks"], z["exps"],
                           log_fn=lambda tag, v, s: logged.append((tag, v, s)))
    got = np.array([[v for tag, v, s in logged if tag == t] for t in
                    ("loss/loss", "loss/value_loss", "loss/surr_loss", "loss/entropy_loss")]).T
    assert got.shape == z["losses"].shape == (epochs * (T // B), 4)
    assert np.allclose(got, z["losses"], rtol=2e-4, atol=2e-5), np.abs(got - z["losses"]).max()
    totals = np.array([out["total_loss"], out["total_value_loss"], out["total_surr_loss"], out["total_entropy_loss"]])
    assert np.allclose(totals, z["totals"], rtol=2e-4, atol=2e-5)
    assert rel(up.flat_params(), z["params_after"]) < 2e-5


def test_batch_stage_groups_minibatches_by_stage():
    """agent_specs.batch_stage (urban_planning_agent.py:273-279,314-319): after the shuffle the states are regrouped
    land-use first, road second, and the update still matches the oracle port driven the same way."""
    from drl_urban_planning_b200.ppo import PPOUpdater
    dev = torch.device("cuda", 0)
    T, B = 48, 16
    states, actions = synth.make_states(43, "small", T)
    spec = synth.COMMUNITIES["small"]
    flat = PL.default_init(43)
    up = PPOUpdater(flat, spec.max_num_nodes, spec.max_num_edges, dev, opt_num_epochs=1, mini_batch_size=B,
                    batch_stage=True)
    up.load_states(states, actions)
    np.random.seed(3)
    order = up._epoch_order(np.arange(T))
    stage = np.array([int(s[8][:2].argmax()) for s in states])
    np.random.seed(3)
    perm = np.arange(T); np.random.shuffle(perm)
    want = np.concatenate([perm[stage[perm] == 0], perm[stage[perm] == 1]])
    assert np.array_equal(order, want)


def test_checkpoint_carries_adam_state(tmp_path):
    """SURVEY 8(f)-4: `use_b200_update` wraps save_checkpoint / load_checkpoint of a reference-shaped agent so that the
    Adam moments travel inside the reference's own pickle under a key it ignores; a resumed run continues the exact
    parameter trajectory (with the first-step clip re-armed like a new reference process, or not)."""
    import pickle
    import types
    from drl_urban_planning_b200.agent import use_b200_update
    from drl_urban_planning_b200.model import ActorCritic, create_sgnn_model
    dev = torch.device("cuda", 0)
    spec = synth.COMMUNITIES["small"]
    T = 32
    states, actions = synth.make_states(61, "small", T)
    rng = np.random.default_rng(61)
    batch = types.SimpleNamespace(states=states, actions=actions, rewards=rng.standard_normal(T).astype(np.float32),
                                  masks=np.ones(T, np.float32), exps=np.ones(T, np.float32))

    def make_agent():
        cfg = Cfg(spec.max_num_nodes, spec.max_num_edges)
        cfg.lr, cfg.eps, cfg.clip_epsilon, cfg.value_pred_coef, cfg.entropy_coef = 4e-4, 1e-5, 0.2, 0.5, 0.01
        cfg.gamma, cfg.tau, cfg.num_optim_epoch, cfg.mini_batch_size, cfg.weightdecay = 1.0, 0.0, 1, 16, 0.0
        cfg.agent_specs, cfg.agent = {}, "rl-sgnn"
        cfg.model_dir, cfg.save_model_interval = str(tmp_path), 1
        ag = Agent()
        ag.cfg, ag.device, ag.loss_iter, ag.tb_logger, ag.save_best_flag, ag.best_rewards = cfg, dev, 0, None, False, 0.0
        torch.manual_seed(9)
        p, v = create_sgnn_model(cfg, ag)
        ag.policy_net, ag.value_net, ag.actor_critic_net = p, v, ActorCritic(p, v)

        def save_checkpoint(iteration):                      # the reference's file format (:172-183)
            cp = {"actor_critic_dict": {k: t.cpu() for k, t in ag.actor_critic_net.state_dict().items()},
                  "loss_iter": ag.loss_iter, "iteration": iteration}
            with open("%s/iteration_%04d.p" % (cfg.model_dir, iteration + 1), "wb") as f:
                pickle.dump(cp, f)

        def load_checkpoint(checkpoint, restore_best_rewards=True):
            cp = pickle.load(open("%s/iteration_%04d.p" % (cfg.model_dir, checkpoint), "rb"))
            ag.actor_critic_net.load_state_dict(cp["actor_critic_dict"])
            ag.loss_iter = cp["loss_iter"]
            return cp["iteration"] + 1
        ag.save_checkpoint, ag.load_checkpoint = save_checkpoint, load_checkpoint
        return ag

    a1 = make_agent()
    c1 = use_b200_update(a1, clip_mode=_lib.CLIP_NEVER)
    np.random.seed(1); a1.update_params(batch, 0)
    a1.save_checkpoint(0)
    cp = pickle.load(open(str(tmp_path / "iteration_0001.p"), "rb"))
    assert "b200_optimizer" in cp and set(cp) >= {"actor_critic_dict", "loss_iter", "iteration"}
    np.random.seed(2); a1.update_params(batch, 1)
    want = c1.updater.flat_params()

    a2 = make_agent()
    c2 = use_b200_update(a2, clip_mode=_lib.CLIP_NEVER)
    assert a2.load_checkpoint(1) == 1
    m1, v1, st1 = (cp["b200_optimizer"][k] for k in ("exp_avg", "exp_avg_sq", "steps"))
    m2, v2, st2 = c2.updater.engine.get_opt_state()
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2) and st1.tolist() == st2.tolist() and st2[0] == 2
    np.random.seed(2); a2.update_params(batch, 1)
    assert np.array_equal(c2.updater.flat_params(), want)        # bit-identical continuation

    a3 = make_agent()                                             # without the moments the trajectory differs
    c3 = use_b200_update(a3, clip_mode=_lib.CLIP_NEVER)
    a3.actor_critic_net.load_state_dict(cp["actor_critic_dict"])
    np.random.seed(2); a3.update_params(batch, 1)
    assert not np.array_equal(c3.updater.flat_params(), want)


def test_dropin_modules_dispatch_to_cuda():
    from drl_urban_planning_b200.model import ActorCritic, create_sgnn_model
    dev = torch.device("cuda", 0)
    spec = synth.COMMUNITIES["small"]
    states, actions = synth.make_states(5, "small", 12)
    torch.manual_seed(3)
    p, v = create_sgnn_model(Cfg(spec.max_num_nodes, spec.max_num_edges), Agent())
    ac = ActorCritic(p, v)
    ts = tensorfy(states)
    with torch.no_grad():
        val_c = v(ts); lp_c, ent_c = p.get_log_prob_entropy(ts, torch.tensor(actions)); gr_c = p.select_action(ts, True)
    ac.to(dev)                                               # to_device(device, actor_critic_net) in the reference
    val_g = v(states)                                        # numpy states: packed, no tensorfy needed
    lp_g, ent_g = p.get_log_prob_entropy([[t.to(dev) for t in s] for s in ts], torch.tensor(actions).to(dev))
    gr_g = p.select_action(states, mean_action=True)
    assert val_g.shape == (12, 1) and val_g.is_cuda
    assert rel(val_g.cpu().numpy(), val_c.numpy()) < 1e-4
    assert rel(lp_g.cpu().numpy(), lp_c.numpy()) < 1e-4 and rel(ent_g.cpu().numpy(), ent_c.numpy()) < 1e-4
    assert np.array_equal(gr_g.cpu().numpy(), gr_c.numpy())
    ac.to("cpu")                                             # to_cpu(policy_net) before forking rollout workers
    assert np.array_equal(p.select_action(ts, True).numpy(), gr_c.numpy())
