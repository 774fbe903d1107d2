"""The deterministic skip-gram kernel (`mvb_sgns_train_det`) over many waves, where a row that one reader of a
wave reads alone is written in place by that reader and every other row goes through the fixed-point
accumulator and the apply.

Every wave but the first of a call runs both paths, so these cases span several waves.  Their exact bits
(tables, loss, pair count) must match digests recorded from the accumulator-only kernel
(tests/golden/record_sgns_det_owner.py), and two of them are checked against an fp64 model of the wave
schedule in which every read sees the tables as the previous wave left them."""
import importlib.util
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def _recorder():
    spec = importlib.util.spec_from_file_location("record_sgns_det_owner",
                                                  os.path.join(GOLDEN, "record_sgns_det_owner.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _sm132():
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("digests and wave sizes are those of a 132-SM H100")


@pytest.mark.parametrize("case", ["zipf_v200k", "uniform_v1m", "hot_v40", "maps_ld320_v100k", "dim37_v100k",
                                  "dim512_w15_k7", "zipf_v200k_2calls"])
def test_sgns_det_owner_bits_match_recorded(mv_device, case):
    with open(os.path.join(GOLDEN, "sgns_det_owner.json")) as f:
        want = json.load(f)["cases"][case]
    _sm132()
    assert _recorder().run_case(case) == want


def _model(case, wave):
    """fp64 model of the wave schedule (tests/sgns_det_model.py): (w_in, w_out) after training, and the rows any
    wave read."""
    spec = importlib.util.spec_from_file_location("sgns_det_model", os.path.join(HERE, "sgns_det_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    r = mod.model(case, wave)
    return r["w_in"], r["w_out"], r["read_in"], r["read_out"]


@pytest.mark.parametrize("case", ["zipf_v200k", "maps_ld320_v100k"])
def test_sgns_det_owner_matches_wave_model(mv_device, case):
    """Tables after training against the fp64 wave model (the bounds of test_gpu_sgns_det_tiles); rows no wave
    read and the pad columns keep their bits, and so does the -0.0 column, whose deltas are all zero."""
    from multiverso_b200 import _native as N
    _sm132()
    rec = _recorder()
    cs = rec.make_case(case)
    c = cs["c"]
    D = c["D"]
    wave = N.cuda_lib().mvb_sgns_win_inflight(D, c["K"], c["W"])
    assert c["n_tok"] > 3 * wave
    w_in, w_out, _, _ = rec.train(cs)
    IN, OUT, read_in, read_out = _model(cs, wave)
    for got, init, ref, read in ((w_in, cs["w_in"], IN, read_in), (w_out, cs["w_out"], OUT, read_out)):
        assert torch.equal(got[:, D:].view(torch.int32), init[:, D:].view(torch.int32))
        assert torch.equal(got[:, 3].view(torch.int32), init[:, 3].view(torch.int32))
        unread = torch.from_numpy(~read)
        assert 0 < int(unread.sum()) < c["V"]
        assert torch.equal(got[unread].view(torch.int32), init[unread].view(torch.int32))
        d_got, d_ref = got[:, :D].double() - init[:, :D].double(), ref - init[:, :D].double()
        err = float(torch.linalg.norm(d_got - d_ref) / torch.linalg.norm(d_ref))
        assert err < 1e-4, err
