"""Run-to-run determinism of the fused MLP-chain kernel under cold weights (regression test of shared-memory races).

The chain kernel streams weight stages through a ring shared by two warpgroups and rewrites each tile's A operand in place
between layers; a stage refilled, or an A row overwritten, before every MMA reading it has completed gives rare, grossly wrong
SDF values of the 9-layer sampling chain.  Such races only show with several tiles per CTA and weight images cold in L2 (as
in a training step, where the backward pass evicts them).  Here: the same launch 200 times with an L2 flush in between,
bit-identical outputs."""
import pytest
import torch

from helpers import build_params

pytestmark = pytest.mark.gpu


def test_sampling_chain_is_bit_reproducible_with_cold_weights():
    from nero_b200.renderer import NeROShapeRenderer
    dev = torch.device('cuda')
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(build_params({}))
    net = net.cuda()
    e = net.engine
    e.prepare_weights()
    rows = 65536                                    # 512 tiles over 132 CTAs: 3-4 tiles per CTA
    e._alloc(1024, 160)
    w = e.w
    g = torch.Generator(device=dev).manual_seed(5)
    X = torch.rand(rows, 64, device=dev, generator=g) - 0.5
    X[:, 39:] = 0
    w['SX0'][:rows].copy_(X)
    w['SC'][:rows, 217:256].copy_(X[:, :39] * 0.70710678)
    out = torch.zeros(rows, 1, device=dev)
    flush = torch.empty(96 * 1024 * 1024, device=dev)       # 384 MB > the 50 MB L2

    def run():
        flush.fill_(1.0)
        e.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], out, None, rows)
        torch.cuda.synchronize()
        return out.clone()

    ref = run()
    assert torch.isfinite(ref).all()
    bad = sum(0 if torch.equal(run(), ref) else 1 for _ in range(200))
    assert bad == 0, f'{bad} of 200 repetitions differ from the first run'
