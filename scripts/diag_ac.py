"""GPU diagnostic: native ActorCritic.predict_act_value forward + backward against torch autograd of the oracle restatement
run on the same GPU in fp32 (TF32 off), one call and short BPTT chains, per-parameter relative errors.
usage: python scripts/diag_ac.py [B ...]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig
    from oracle import torch_oracle as O

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    cfg = O.ActorCriticCfg()
    sd = O.seeded_actor_critic_state_dict(cfg, 556)
    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    ac.load_state_dict(sd)
    ac = ac.to(dev).train()
    batches = [int(a) for a in sys.argv[1:]] or [4, 1, 32]
    for b in batches:
        for steps in (1, 3):
            g = torch.Generator().manual_seed(10 * b + steps)
            obs = [(torch.rand(b, 3, 64, 64, generator=g) * 2 - 1).to(dev) for _ in range(steps)]
            hx0 = (torch.randn(b, cfg.lstm_dim, generator=g) * 0.3).to(dev)
            cx0 = (torch.randn(b, cfg.lstm_dim, generator=g) * 0.3).to(dev)
            gl = [torch.randn(b, cfg.num_actions, generator=g).to(dev) for _ in range(steps)]
            gv = [torch.randn(b, generator=g).to(dev) for _ in range(steps)]

            def run(fn):
                hx, cx = hx0.clone(), cx0.clone()
                loss = 0
                for t in range(steps):
                    logits, val, (hx, cx) = fn(obs[t], hx, cx)
                    loss = loss + (logits * gl[t]).sum() + (val * gv[t]).sum()
                loss = loss + 0.1 * hx.sum() + 0.05 * cx.sum()
                return loss

            # oracle on the GPU (fp32)
            sdd = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
            ref_loss = run(lambda o, h, c: O.predict_act_value(o, h, c, sdd, cfg))
            ref_loss.backward()
            for p in ac.parameters():
                p.grad = None
            loss = run(lambda o, h, c: ac.predict_act_value(o, (h, c)))
            loss.backward()
            torch.cuda.synchronize()
            num = den = 0.0
            rows = []
            for k, p in ac.named_parameters():
                r = sdd[k].grad.double()
                d = p.grad.double() - r
                num += float(d.pow(2).sum()); den += float(r.pow(2).sum())
                rows.append((k, float(d.norm() / r.norm().clamp_min(1e-30)), float(r.norm())))
            print(f"B={b} steps={steps}: "
                  f"loss {float(loss):.6f} ref {float(ref_loss):.6f}  whole-grad rel err {(num / den) ** 0.5:.3e}", flush=True)
            if b == batches[0]:
                for k, e, n in rows:
                    print(f"     {e:9.3e} |g|={n:9.3e} {k}")


if __name__ == "__main__":
    main()
