"""GPU, world_size 2: DD-PPO's exchange on the CUDA path -- the port of the reference's
test/test_ddppo_reduce.py:28-132 (gradients / parameters equal across ranks after the reduce) plus the checks
DDP cannot make: the reduced gradient equals the single-process mean of the rank gradients, the packed
RunningMeanAndVar all-reduce leaves identical running statistics on every rank, and `before_step` produces the same
parameters a single process gets from the averaged gradient.

Two processes are spawned, one GPU each, NCCL backend (what the bench runs): the test needs >= 2 visible GPUs and is
SKIPPED on a 1-GPU machine -- two processes time-slicing one GPU with persistent / cooperative kernels is not a
configuration the path supports.  The file name
sorts last so that, whatever happens here, every other GPU test has already run.  bench.py asserts the same
cross-rank equality after its timed steps at N = 2 / 4 / 8 (`cross_rank_equality` in the JSON line)."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, ngpu, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank if ngpu >= world else 0)
    torch.cuda.set_device(dev)
    if ngpu >= world:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import habitat_lab_b200 as hb
        from habitat_lab_b200.synthetic import fill_rollout_, pointnav_spaces

        hb.load()
        T, N = 8, 4
        obs_space, act_space = pointnav_spaces(128, 128)
        torch.manual_seed(1234 + 17 * rank)   # DIFFERENT initial weights per rank: init_distributed must broadcast rank 0's
        pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=2, rnn_type="LSTM",
                                      normalize_visual_inputs=True).to(dev)
        pol.train()
        ppo = hb.DDPPO(pol, clip_param=0.2, ppo_epoch=1, num_mini_batch=1, value_loss_coef=0.5, entropy_coef=0.01,
                       lr=2.5e-4, eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True,
                       use_normalized_advantage=True)
        ppo.init_distributed(find_unused_params=False)
        flat = pol.flatten_parameters_()
        p0 = flat["params"].detach().clone()
        st = hb.RolloutStorage(T, N, obs_space, act_space, pol)
        st.to(dev)
        nv = fill_rollout_(st, seed=50 + rank, p_done=0.1)   # different rollouts per rank
        st.compute_returns(nv, True, 0.99, 0.95)
        adv = ppo.get_advantages(st)                        # distributed var/mean: one packed all-reduce
        torch.manual_seed(7)
        batch = next(iter(st.data_generator(adv, 1)))
        hook, pol.tail_grads_hook = pol.tail_grads_hook, None   # step 1: the plain path, so the LOCAL gradients can be read
        pol.loss_and_backward(batch, 0.2, 0.5, 0.01, True)   # includes the packed RunningMeanAndVar all-reduce
        g_local = flat["grads"].detach().clone()
        gn = float(ppo.before_step())                         # all-reduce + clip + Adam (the code under test); the
        torch.cuda.synchronize()                              # returned tensor is a reused device scalar: read it now
        stats = torch.cat([b.detach().flatten().double() for b in pol.buffers()])
        g_red, p_after = flat["grads"].detach().cpu().numpy(), flat["params"].detach().cpu().numpy()
        # step 2: the overlapped path -- the recurrent / head chunk is reduced from inside the backward pass
        assert hook is not None, "DDPPO.init_distributed must install the tail-gradient hook"
        pol.tail_grads_hook = hook
        pol.loss_and_backward(batch, 0.2, 0.5, 0.01, True)
        ppo.before_step()
        torch.cuda.synchronize()
        p_after2 = flat["params"].detach().cpu().numpy()
        q.put((rank, p0.cpu().numpy(), g_local.cpu().numpy(), g_red, p_after, gn, stats.cpu().numpy(),
               adv.detach().cpu().numpy(), st.buffers["returns"].cpu().numpy(), st.buffers["value_preds"].cpu().numpy(),
               p_after2))
    except BaseException:   # report instead of leaving the parent waiting on the queue
        import traceback
        q.put(("error", rank, traceback.format_exc()[-3000:]))
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_ddppo_before_step_two_ranks(hb):
    from oracle import torch_oracle as O

    world = 2
    ngpu = torch.cuda.device_count()
    if ngpu < world:
        pytest.skip("needs >= 2 GPUs (one rank per GPU, NCCL)")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, ngpu, q)) for r in range(world)]
    [p.start() for p in procs]
    res = []
    import queue as _queue
    import time as _time
    deadline = _time.time() + 420
    try:
        while len(res) < world:
            try:
                item = q.get(timeout=5)
            except _queue.Empty:
                dead = [p.exitcode for p in procs if p.exitcode not in (None, 0)]
                assert not dead, f"a rank died with exit code {dead} before reporting"
                assert _time.time() < deadline, "ranks did not finish in time"
                continue
            assert item[0] != "error", f"rank {item[1]} failed:\n{item[2]}"
            res.append(item)
    finally:
        for p in procs:
            p.join(20)
            if p.is_alive():
                p.kill()
    res.sort(key=lambda t: t[0])
    r0, r1 = [[torch.from_numpy(a) if hasattr(a, "shape") else a for a in r] for r in res]
    # 1. broadcast: both ranks start from rank 0's weights although they were initialised with different seeds
    assert torch.equal(r0[1], r1[1])
    # 2. test_ddppo_reduce.py:111-118 -- the reduced gradients are equal on every rank ...
    assert torch.equal(r0[3], r1[3])
    # ... and equal to the single-process SUM of the rank gradients (the 1/world mean is folded into the Adam kernel)
    assert (r0[2] - r1[2]).abs().max().item() > 0, "ranks must see different data"
    torch.testing.assert_close(r0[3], r0[2] + r1[2], rtol=1e-6, atol=1e-9)
    # 3. parameters after the step are bit-identical across ranks, and what a single process computes from the mean
    assert torch.equal(r0[4], r1[4])
    mean_g = ((r0[2].double() + r1[2].double()) / 2).float()
    assert r0[5] == pytest.approx(mean_g.double().norm().item(), rel=1e-5)
    p, m, v = r0[1].clone(), torch.zeros_like(r0[1]), torch.zeros_like(r0[1])
    O.clip_adam_step([p], [mean_g], [m], [v], 1, 2.5e-4, (0.9, 0.999), 1e-5, 0.2)
    torch.testing.assert_close(r0[4], p, rtol=1e-5, atol=2e-7)
    # 3b. second step through the overlapped exchange (tail chunk all-reduced during the encoder backward): still identical
    assert torch.equal(r0[10], r1[10]) and torch.isfinite(r0[10]).all() and not torch.equal(r0[10], r0[4])
    # 4. RunningMeanAndVar buffers (synced by the packed statistics all-reduce) identical on both ranks
    assert torch.equal(r0[6], r1[6])
    assert r0[6][-1].item() == 2 * 32, "count = frames of both ranks (T*N each)"
    # 5. normalised advantages used the GLOBAL mean / variance (ddppo.py:59-84; statistics over the whole buffers)
    var, mean = O.distributed_var_mean([(r[8] - r[9]).flatten() for r in (r0, r1)])
    for r in (r0, r1):
        torch.testing.assert_close(r[7][:8], O.get_advantages(r[8], r[9], True, var_mean=(var, mean))[:8],
                                   rtol=1e-4, atol=1e-5)
