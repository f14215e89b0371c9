"""The configurations bench.py times, against the unmodified reference's outputs (tests/golden/full_cfg2/3/5, checked by
oracle/full_golden.py per view, per border line and per output).

bench.py times CUDA-graph replays, so for cfg2, cfg3 and cfg5, and for the 392 x 518 and 882 x 518 inputs of
full_land_s10 and full_tall_s3, the replay (third call of a signature) must equal the eager forward bit for bit and pass the
same bars.  cfg4 runs several scenes per forward call: the full_cfg2 inputs as scene 3 of a
B = 4 call must give what the reference gives for them alone."""
import pytest
import torch

from oracle import full_golden
from oracle.synth import make_inputs
from test_model_gpu import FULL_INDEX, KEYS, full_model, full_size_check, set_heads

pytestmark = pytest.mark.gpu


def _inputs(meta, B=1, seed=None):
    return make_inputs(B, meta["S"], meta["H"], meta["W"], seed=meta["input_seed"] if seed is None else seed)


@pytest.mark.parametrize("case", ["full_cfg2", "full_cfg3", "full_cfg5", "full_land_s10", "full_tall_s3"])
def test_full_size_graph_replay_matches_eager_and_reference(case):
    meta = FULL_INDEX[case]
    m = full_model()
    set_heads(m, "fp16")
    m.use_cuda_graph = True
    m._graphs = {}
    inp = {k: v.cuda() for k, v in _inputs(meta).items()}
    kw = dict(depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"])
    try:
        eager = m(**inp, **kw)
        m(**inp, **kw)
        replay = m(**inp, **kw)                    # captured, then replayed
        torch.cuda.synchronize()
        assert len(m._graphs) == 1 and next(iter(m._graphs.values()))["graph"] is not None, "graph was not captured"
    finally:
        m._graphs = {}                            # the graph's private pool holds a 24-view forward's outputs
        torch.cuda.empty_cache()
    for k in KEYS:
        assert torch.equal(replay[k], eager[k]), k
    for i in range(4):
        assert torch.equal(replay["pose_enc_list"][i], eager["pose_enc_list"][i]), i
    full_size_check(case, replay, "heads=fp16 graph replay")


def test_full_size_scene_batch_of_four():
    """cfg4 shape: B = 4 scenes x 8 views, images only; the full_cfg2 inputs are scene 3, seeded scenes fill slots 0..2."""
    meta = FULL_INDEX["full_cfg2"]
    assert meta["depth_gt_index"] == [] and meta["camera_gt_index"] == []
    m = full_model()
    set_heads(m, "fp16")
    others, mine = _inputs(meta, B=3, seed=101), _inputs(meta)
    inp = {k: torch.cat([others[k], mine[k]]).cuda() for k in mine}
    out = m(depth_gt_index=[], camera_gt_index=[], **inp)
    torch.cuda.synchronize()
    assert out["depth"].shape == (4, meta["S"], meta["H"], meta["W"], 1)
    scene3 = {k: out[k][3:4] for k in KEYS}
    scene3["pose_enc_list"] = [p[3:4] for p in out["pose_enc_list"]]
    full_size_check("full_cfg2", scene3, "heads=fp16 scene 3 of B=4")
    del out
    torch.cuda.empty_cache()
