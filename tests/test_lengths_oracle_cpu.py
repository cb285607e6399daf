"""CPU checks of oracle/lengths_oracle.py: with every length equal to T it is the existing oracle (OracleBiGRU with the
same parameters) in logits, h_n and every gradient; with shorter lengths each row is the unpadded model run on its own
prefix, and padded inputs have no effect."""
import pytest
import torch

from oracle.bigru_oracle import OracleBiGRU
from oracle.lengths_oracle import LengthsOracle


def _models(H, F, C, L, D, seed=0):
    torch.manual_seed(seed)
    ref = OracleBiGRU(H, F, C, L, 50, 0.0, False, D == 2).double().eval()
    return ref, LengthsOracle(ref.state_dict(), H, F, L, D == 2)


@pytest.mark.parametrize("L,D", [(1, 2), (2, 2), (3, 1)])
def test_full_lengths_equal_existing_oracle(L, D):
    B, T, F, H, C = 5, 7, 6, 9, 3
    ref, orc = _models(H, F, C, L, D)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, F, generator=g, dtype=torch.float64)
    dl = torch.randn(B, C, generator=g, dtype=torch.float64)
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    want = ref(xa)
    _, hn_want = ref.gru(x)
    got, hn, _ = orc(xb, [T] * B)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(hn, hn_want, rtol=1e-12, atol=1e-12)
    want.backward(dl)
    got.backward(dl)
    torch.testing.assert_close(xb.grad, xa.grad, rtol=1e-12, atol=1e-12)
    gref = torch.cat([p.grad.reshape(-1) for p in
                      [getattr(ref.gru, f"{n}_l{l}{'_reverse' if d else ''}") for l in range(L) for d in range(D)
                       for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")] + [ref.linear.weight, ref.linear.bias]])
    torch.testing.assert_close(orc.flat_grads(), gref, rtol=1e-12, atol=1e-12)


def test_short_rows_are_their_own_prefix():
    """Row b with length n gives the logits and input gradient of the unpadded model on x[b, :n]; padded inputs are
    ignored (whatever they hold) and get a zero gradient."""
    B, T, F, H, C, L = 4, 6, 5, 7, 3, 2
    ref, orc = _models(H, F, C, L, 2, seed=3)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, T, F, generator=g, dtype=torch.float64)
    lens = [1, 6, 3, 4]
    noisy = x.clone()
    for b, n in enumerate(lens):
        noisy[b, n:] = 1e3 * torch.randn(T - n, F, generator=g, dtype=torch.float64)
    xg = noisy.clone().requires_grad_(True)
    got, _, _ = orc(xg, lens)
    got.sum().backward()
    for b, n in enumerate(lens):
        xb = x[b:b + 1, :n].clone().requires_grad_(True)
        want = ref(xb)
        torch.testing.assert_close(got[b:b + 1], want, rtol=1e-12, atol=1e-12)
        want.sum().backward()
        torch.testing.assert_close(xg.grad[b, :n], xb.grad[0], rtol=1e-10, atol=1e-12)
        assert (xg.grad[b, n:] == 0).all()
