"""The diamond_b200:: custom ops behind WorldModelEnv.predict_next_obs / predict_rew_end, without a GPU: their schemas declare
the mutations, the fake kernels give the eager results' shapes, dtypes and aliasing, eager calls reach the same C entry points
(a stand-in library records them), and both methods trace whole under torch.compile(fullgraph=True) (native bodies stubbed)."""
import types

import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from diamond_b200 import _lib, torch_ops
from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, DiffusionSampler, DiffusionSamplerConfig, InnerModelConfig
from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
from diamond_b200.synthetic import frame_stacks

B, S, D = 4, 16, 32


def _models():
    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 64, [1, 1], [32, 32], [0, 0], 4), 0.5, 0.3)).eval()
    rem = RewEndModel(RewEndModelConfig(D, 3, S, 32, [1, 1], [32, 32], [0, 0], 4)).eval()
    return den, rem


def _writes(op):
    return {a.name for a in op.default._schema.arguments if a.alias_info is not None and a.alias_info.is_write}


def test_ops_are_registered_with_their_mutations():
    assert _writes(torch.ops.diamond_b200.sample_ring) == {"frames", "traj", "workspace"}
    assert _writes(torch.ops.diamond_b200.rew_end_predict) == {"workspace"}
    assert len(torch.ops.diamond_b200.sample_ring.default._schema.returns) == 0
    assert len(torch.ops.diamond_b200.rew_end_predict.default._schema.returns) == 4
    names = [a.name for a in torch.ops.diamond_b200.sample_ring.default._schema.arguments]
    assert names[0] == "key" and names[-1] == "params"


def test_fake_kernels_match_eager_results():
    _, rem = _models()
    key = torch_ops.key_of(rem)
    with FakeTensorMode():
        obs, nxt = torch.empty(B, 3, 3, S, S), torch.empty(B, 3, 3, S, S)
        act, hx, cx, ws = torch.empty(B, 3, dtype=torch.long), torch.empty(B, D), torch.empty(B, D), torch.empty(64, dtype=torch.uint8)
        outs = torch.ops.diamond_b200.rew_end_predict(key, obs, act, nxt, hx, cx, ws, [])
        assert [tuple(o.shape) for o in outs] == [(B, 3, 3), (B, 3, 2), (B, D), (B, D)]
        assert all(o.dtype == torch.float32 for o in outs)
        ins = (obs, act, nxt, hx, cx, ws)
        assert not any(o.untyped_storage()._cdata == i.untyped_storage()._cdata for o in outs for i in ins)
        frames, acts, traj = torch.empty(4, B, 3, S, S), torch.empty(4, B, dtype=torch.long), torch.empty(4, B, 3, S, S)
        assert torch.ops.diamond_b200.sample_ring(key, frames, acts, 1, traj, None, ws, []) is None


class _RecordingLib:
    def __init__(self):
        self.calls = []

    def dmd_sampler_sample(self, h, sc, b, hh, ww, obs, act, head, traj, eps, out, ws, ws_bytes, graph, stream):
        self.calls.append(("dmd_sampler_sample", h, b, hh, ww, obs, act, head, traj, out, ws))
        return 0

    def dmd_rew_end_predict(self, h, b, t, obs, nxt, act, hx, cx, rew, end, hx_o, cx_o, ws, ws_bytes, stream):
        self.calls.append(("dmd_rew_end_predict", h, b, t, obs, nxt, act, hx, cx, ws))
        return 0


def test_eager_calls_reach_the_same_entry_points(monkeypatch):
    fake = _RecordingLib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    den, rem = _models()
    den.inner_model.native = lambda *a: 7
    rem._native = lambda: 9
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(3))
    sampler._ws_bytes[(B, S, S, torch.are_deterministic_algorithms_enabled())] = 256
    rem._ws_bytes = {(B * 2, torch.are_deterministic_algorithms_enabled()): 128}

    frames, acts = torch.zeros(4, B, 3, S, S), torch.zeros(4, B, dtype=torch.long)
    traj = sampler.sample_ring(frames, acts, 2)
    name, h, b, hh, ww, obs, act, head, traj_p, out, ws = fake.calls[-1]
    assert (name, h, b, hh, ww, head) == ("dmd_sampler_sample", 7, B, S, S, 2)
    assert (obs, act, traj_p, out) == (frames.data_ptr(), acts.data_ptr(), traj.data_ptr(), frames[2].data_ptr())
    assert ws == den.inner_model._ws.data_ptr()

    o, n, a = torch.zeros(B, 2, 3, S, S), torch.zeros(B, 2, 3, S, S), torch.zeros(B, 2, dtype=torch.long)
    hx, cx = torch.zeros(1, B, D), torch.zeros(1, B, D)
    with torch.no_grad():
        rew, end, (hx_o, cx_o) = rem.predict_rew_end(o, a, n, (hx, cx))
    name, h, b, t, obs, nxt, act, hx_p, cx_p, ws = fake.calls[-1]
    assert (name, h, b, t) == ("dmd_rew_end_predict", 9, B, 2)
    assert (obs, nxt, act, hx_p, cx_p, ws) == (o.data_ptr(), n.data_ptr(), a.data_ptr(), hx.data_ptr(), cx.data_ptr(), rem._ws.data_ptr())
    assert rew.shape == (B, 2, 3) and end.shape == (B, 2, 2) and hx_o.shape == cx_o.shape == (1, B, D)
    assert len(fake.calls) == 2


def test_world_model_methods_trace_whole():
    """predict_next_obs and predict_rew_end compile with fullgraph=True (aot_eager on the CPU; the native bodies are replaced
    by torch stand-ins), over several ring heads and through reset_dead's burn-in."""
    den, rem = _models()
    pool = [frame_stacks(B, 4, 3, S, S, 4, k)[:2] for k in range(4)]

    class Loader:
        batch_sampler = types.SimpleNamespace(batch_size=B)

        def __iter__(self):
            k = 0
            while True:
                obs, act = pool[k % len(pool)]
                k += 1
                yield types.SimpleNamespace(obs=obs, act=act)

    env = WorldModelEnv(den, rem, Loader(), WorldModelEnvConfig(3, 2, DiffusionSamplerConfig(3)))
    calls = []

    def sample(frames, acts, head, traj, eps, out, ws):
        calls.append("sample")
        t = frames.size(0)
        traj[1:].copy_(traj[0] * 0.5 + frames[(head + t - 1) % t] * 0.5)
        out.copy_(traj[-1])

    def predict(obs, act, nxt, hx, cx, ws):
        calls.append("predict")
        f = obs.flatten(2).mean(-1) + nxt.flatten(2).mean(-1)
        h = (hx if hx is not None else torch.zeros(obs.size(0), D)) + f[:, -1:]
        return torch.stack([f, -f, f], -1), torch.stack([f * 0 + 4, f], -1), h.clone(), h * 0.5

    env.sampler._sample_native = sample
    rem._predict_native = predict
    rem._native = lambda: None
    env.sampler._ws_bytes[(B, S, S, False)] = 256
    rem._ws_bytes = {(B, False): 128, (B * 3, False): 128}
    den.inner_model._state_tensors(), rem._state_tensors()
    env.predict_next_obs = torch.compile(env.predict_next_obs, backend="aot_eager", fullgraph=True)
    env.predict_rew_end = torch.compile(env.predict_rew_end, backend="aot_eager", fullgraph=True)
    torch._dynamo.reset()
    try:
        env.reset()
        hx_buf = env.hx_rew_end
        for _ in range(7):
            obs, rew, end, trunc, info = env.step(torch.randint(0, 4, (B,)))
        assert trunc.all() or "burnin_obs" in info or env.ep_len.max() < 3
        assert env.hx_rew_end is hx_buf                    # the carried state stays in its static buffer
        assert calls.count("sample") == 7 and calls.count("predict") >= 7
    finally:
        torch._dynamo.reset()
