"""Every drop-in model's cal_loss + backward and full_predict on the GPU against the oracle in float64, on the contraction
and propagation paths the golden shapes (d = 32 / 64, tau 0.1-0.2) never select: the FP32-FMA InfoNCE contraction at
d = 16, 20, 48, 128, propagation at d = 4, the 3xTF32 contraction at tau = 0.05, both sides of the 3xFP16 offset bound,
and HCCF's hyper branch at other (d, hyper_num).  The graph (600 users x 450 items with a split hub row on each side and
isolated rows) and the ragged batch are built by ``ssl_test_helpers.path_case``; tests/test_host_model_paths.py shows on
the host that the float32 oracle meets the bounds used here and that slightly wrong ones do not.

Each case records which contraction entry points of the library ran and asserts the one its row names."""
import numpy as np
import pytest
import torch

import ssl_test_helpers as H

pytestmark = pytest.mark.gpu


class _Recorder:
    """Stands in for ``engine.lib``: the names of the InfoNCE contraction / pairwise-uniformity entry points called."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not (name.startswith('ssl_softmax_gemm') or name == 'ssl_uniform_pairs'):
            return fn

        def rec(*args):
            self.calls.append(name)
            return fn(*args)
        return rec


def _record(monkeypatch):
    from sslrec_b200 import engine
    rec = _Recorder(engine.lib)
    monkeypatch.setattr(engine, 'lib', rec)
    return rec


def _expected(model_key, dim, tau, batch, live=False):
    """The contraction a case must run: the FFMA kernel at d not in {32, 64}, 3xTF32 below tau = 0.0902 (offset log2(e) / tau
    above 16), else 3xFP16; LightGCL's raw rows always take 3xTF32 on tensor cores; DirectAU sums its uniformity pairs
    directly below 256 rows.  ``live``: the device-count-bounded variant (HCCF under a CUDA graph)."""
    name = model_key.split('_')[0]
    if name == 'lightgcn':
        return set()
    if name == 'directau' and batch < 256:
        return {'ssl_uniform_pairs'}
    if dim not in (32, 64):
        fn = 'ssl_softmax_gemm'
    elif name == 'lightgcl' or tau < 0.0902:
        fn = 'ssl_softmax_gemm_tf32x3'
    else:
        fn = 'ssl_softmax_gemm_f16x3'
    return {fn + ('_live' if live else '')}


def _gpu_model(model_key, case, hp, adj, dr, st, inject=True):
    """The model on the oracle's parameters; ``inject``: also its draws and NCL's k-means state."""
    model, _ = H.make_model(model_key, case, hp, inject=H.gpu_injection(model_key, case, hp, adj, dr) if inject else None)
    model.load_state_dict({k: v.detach() for k, v in H.path_params(model_key, case, dr, torch.float32).items()})
    if model_key == 'lightgcl':
        model.ut, model.vt, model.u_mul_s, model.v_mul_s = (torch.from_numpy(st['svd_' + k]).cuda() for k in ('ut', 'vt', 'u_mul_s', 'v_mul_s'))
    if model_key == 'ncl' and inject:
        for k in ('user_centroids', 'item_centroids', 'user2cluster', 'item2cluster'):
            setattr(model, k, torch.from_numpy(st[k]).cuda())
    return model


def _batch(model_key, ancs, poss, negs):
    b = [torch.from_numpy(np.asarray(a)).long().cuda() for a in (ancs, poss, negs)]
    if model_key == 'ncl':
        b.append(torch.zeros(len(ancs), dtype=torch.int64, device='cuda'))          # no re-clustering flag
    return b


@pytest.mark.parametrize('model_key,dim,tau,batch,hyper_num', H.PATH_CASES, ids=[H.path_case_id(c) for c in H.PATH_CASES])
def test_model_matches_float64(model_key, dim, tau, batch, hyper_num, monkeypatch):
    case, hp, adj, dr, st = H.path_setup(model_key, dim, tau, batch, hyper_num)
    margin = H.kink_margin(model_key, case, hp, adj, dr, st)
    assert margin > H.KINK_MARGIN, f'ill-posed case: a kink input within {margin:.2e} of its |term| sum'
    ref = H.path_oracle(model_key, case, hp, adj, dr, st, torch.float64)

    model = _gpu_model(model_key, case, hp, adj, dr, st)
    rec = _record(monkeypatch)
    loss, parts = model.cal_loss(_batch(model_key, case['ancs'], case['poss'], case['negs']))
    loss.backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    got = dict(loss=loss.item(), parts={k: float(v) for k, v in parts.items()},
               grads={k: p.grad.double().cpu().numpy() for k, p in model.named_parameters()})
    users, mask = H.pred_users_mask(case)
    model.eval()
    with torch.no_grad():
        got['preds'] = model.full_predict([users.cuda(), mask.cuda()]).double().cpu().numpy()

    errs = H.path_errors(got, ref)
    worst = max(errs, key=errs.get)
    print(f'{H.path_case_id((model_key, dim, tau, batch, hyper_num))}: largest error {errs[worst]:.3f} of its bound ({worst}); '
          f'contraction {sorted(set(rec.calls))}')
    assert set(rec.calls) == _expected(model_key, dim, tau, batch), rec.calls
    assert errs[worst] <= 1.0, errs


GRAPH_CASES = [('hccf', 48, 0.2), ('ncl', 48, 0.2), ('hccf', 32, 0.05), ('ncl', 32, 0.05)]


@pytest.mark.parametrize('model_key,dim,tau', GRAPH_CASES)
def test_graphed_step_equals_eager_step(model_key, dim, tau, monkeypatch):
    """One GraphedStep replay equals the eager step on the same batch after the same two warm-up steps (HCCF's eager loop on
    its graph-safe path), through the FFMA and 3xTF32 contractions: HCCF's spec-node terms run ``ssl_softmax_gemm_live`` /
    ``ssl_softmax_gemm_tf32x3_live`` there."""
    from sslrec_b200.graphed import GraphedStep
    from sslrec_b200.optim import FusedAdam
    hccf = model_key == 'hccf'
    case, hp, adj, dr, st = H.path_setup(model_key, dim, tau, 300, None)
    rs = np.random.RandomState(3)
    pick = rs.randint(0, len(case['rows']), size=case['batch'])
    batches = [_batch(model_key, case['ancs'], case['poss'], case['negs']),
               _batch(model_key, case['rows'][pick], case['cols'][pick], rs.randint(0, case['n_item'], size=case['batch']))]
    out = {}
    for mode in ('eager', 'graph'):
        torch.manual_seed(0)            # same parameter init and the same generator for NCL's k-means in both runs
        np.random.seed(0)
        model = _gpu_model(model_key, case, hp, adj, dr, st, inject=False)      # in-kernel draws; NCL clusters on its first step
        opt = FusedAdam(model.parameters(), lr=1e-2)
        rec = _record(monkeypatch)
        if mode == 'eager':
            model._graph_mode = hccf
            for b in (batches[0], batches[0], batches[1]):
                opt.zero_grad()
                loss, _ = model.cal_loss(b)
                loss.backward()
                opt.step()
            model._graph_mode = False
        else:
            step = GraphedStep(model, opt, batches[0], warmup=2)
            loss, _ = step(batches[1])
            step.close()
        last = loss.item()
        monkeypatch.undo()
        assert set(rec.calls) == _expected(model_key, dim, tau, 300, live=hccf), (mode, sorted(set(rec.calls)))
        out[mode] = (last, torch.cat([p.detach().reshape(-1) for p in model.parameters()]).clone())
    (lg, pg), (le, pe) = out['graph'], out['eager']
    print(f'{model_key}-d{dim}-tau{tau}: graph loss {lg:.8f} eager {le:.8f}, max |d param| {(pg - pe).abs().max().item():.2e}')
    assert abs(lg - le) <= 1e-6 * max(1.0, abs(le)), (lg, le)
    assert torch.allclose(pg, pe, rtol=1e-5, atol=3e-4), (pg - pe).abs().max().item()
