"""CUDA-graph capture next to other host threads.  `TiledModel._graphed` captures a forward's first call at each key, and
`Tester.run` keeps a PNG writer thread that waits on the previous image's device-to-host copy events meanwhile.  The
capture must bar only its own thread from unsafe CUDA calls: a wait on an event in another thread must neither fail
nor invalidate the capture."""
import threading

import pytest
import torch

from test_baseline_host import pretrain_model_cfg

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def test_event_wait_in_another_thread_during_capture(cuda):
    from patchfusion_b200.baseline import BaselinePretrain
    cfg = pretrain_model_cfg('vits', 'coarse')
    cfg.pop('type')
    model = BaselinePretrain(**cfg).init_synthetic_weights(0).to(cuda).eval()
    lr = torch.rand(2, 3, 392, 518, generator=torch.Generator().manual_seed(5)).to(cuda)
    model.use_cuda_graphs = False
    want = model(mode='infer', image_lr=lr, image_hr=None)[0].clone()
    model.use_cuda_graphs = True
    # a copy on a side stream and its event, as Tester._emit records them
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        host = torch.empty(1 << 20, dtype=torch.float32).pin_memory()
        host.copy_(torch.ones(1 << 20, device=cuda), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(side)
    eng = model.engine((392, 518))
    branch, waits, errors = eng.branch, [], []

    def wait():
        try:
            ev.synchronize()
            waits.append(torch.cuda.is_current_stream_capturing())
        except Exception as e:       # noqa: BLE001 - reported below
            errors.append(repr(e))

    def branch_with_waiter(*a, **kw):
        if torch.cuda.is_current_stream_capturing():
            t = threading.Thread(target=wait)
            t.start()
            t.join()
        return branch(*a, **kw)
    eng.branch = branch_with_waiter
    try:
        y0 = model(mode='infer', image_lr=lr, image_hr=None)[0].clone()     # eager pass + capture
    finally:
        del eng.branch
    assert errors == [] and waits == [False], (errors, waits)
    assert ('coarse', 2, 392, 518) in model._graphs
    y1 = model(mode='infer', image_lr=lr, image_hr=None)[0].clone()         # replay
    assert torch.equal(y0, want) and torch.equal(y1, want)
    assert (host == 1).all()
