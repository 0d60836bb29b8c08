"""CPU checks of VirConv8x's static-mode front end and the two-stream bookkeeping of graph.GraphedStep / executor: what is
refused, and with which error, before anything reaches a device."""
import pytest
import torch

CFG8 = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])


def _spec():
    from virconv_b200 import executor
    return executor.StaticSpec(torch.zeros(1, dtype=torch.int32), {}, torch.zeros(1, dtype=torch.int32))


def _bd(**extra):
    bd = {'voxel_features': torch.zeros(4, 8), 'voxel_coords': torch.zeros(4, 4), 'voxel_features_mm': torch.zeros(4, 8),
          'voxel_coords_mm': torch.zeros(4, 4), 'batch_size': 2, 'calib': None, 'virconv_proj': torch.zeros(2, 28)}
    bd.update(extra)
    return bd


def _model(cfg=CFG8, **kw):
    from virconv_b200.backbone import VirConv8x
    return VirConv8x(cfg, 8, [1408, 1600, 80], **kw)


def test_eval_forward_with_static_spec_raises():
    m = _model().eval()
    with pytest.raises(ValueError, match='training forward only'):
        m(_bd(virconv_static=_spec(), virconv_static_mm=_spec()))
    with pytest.raises(ValueError, match='training forward only'):
        m(_bd(virconv_static=_spec(), virconv_static_mm=_spec(), transform_param=torch.zeros(2, 3, 3)))


def test_static_training_forward_refusals():
    m = _model().train()
    with pytest.raises(ValueError, match="virconv_static_mm"):
        m(_bd(virconv_static=_spec()))                                   # one stream without its spec
    with pytest.raises(ValueError, match='one copy per stream'):
        m(_bd(virconv_static=_spec(), virconv_static_mm=_spec(), transform_param=torch.zeros(2, 3, 3)))
    with pytest.raises(ValueError, match='virconv_proj'):
        m(_bd(virconv_static=_spec(), virconv_static_mm=_spec(), virconv_proj=None))
    phased = _spec()
    phased.phase = 1
    with pytest.raises(ValueError, match='VirConvL8x only'):
        m(_bd(virconv_static=_spec(), virconv_static_mm=phased))
    host = _model(discard_mode='paper', discard_rng='numpy').train()
    with pytest.raises(ValueError, match='no static form'):
        host(_bd(virconv_static=_spec(), virconv_static_mm=_spec()))
    dev = _model(discard_mode='paper', discard_rng='device').train()
    with pytest.raises(ValueError, match='no static form'):
        dev(_bd(virconv_static=_spec(), virconv_static_mm=_spec(), stvd_keep_rows=[[0]] * 4))
    lidar_only = _model(dict(CFG8, MM=False)).train()
    assert lidar_only.static_streams == ('',)
    with pytest.raises(ValueError, match="virconv_static'"):
        lidar_only(_bd(virconv_static=_spec(), virconv_static_mm=_spec()))


def test_streams_of_graphed_and_pipelined_steps():
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import GraphedStep, PipelinedStep
    m = _model()
    assert m.static_streams == ('', '_mm')
    assert [(st.sfx, st.i) for st in GraphedStep(m, None).streams] == [('', 0), ('_mm', 1)]
    assert [st.sfx for st in GraphedStep(VirConvL8x(CFG, 8, [1408, 1600, 80]), None).streams] == ['']
    with pytest.raises(ValueError, match='PipelinedStep.*GraphedStep'):
        PipelinedStep(m, None)
    # per-stream voxeliser settings: `_mm` entries where given; the MM stream's VFE is the plain mean by default
    vox = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
               max_voxels=16000, vfe_model='max')
    g = GraphedStep(m, None, voxelizer=vox)
    lidar, mm = g.streams
    assert (g._vox_arg(lidar, 'max_voxels'), g._vox_arg(lidar, 'vfe_model')) == (16000, 'max')
    assert (g._vox_arg(mm, 'max_voxels'), g._vox_arg(mm, 'vfe_model')) == (16000, None)
    g = GraphedStep(m, None, voxelizer=dict(vox, max_voxels_mm=8000, vfe_model_mm='max'))
    assert (g._vox_arg(g.streams[1], 'max_voxels'), g._vox_arg(g.streams[1], 'vfe_model')) == (8000, 'max')
    assert g._vox_arg(g.streams[0], 'max_voxels') == 16000


class _FakeRun:
    """What executor.RunCounts reads of a run record: the plan's rulebooks and an index-set query."""

    class _Plan:
        rb_keys = {0: ((), 3, 0, 0), 1: ((), 3, 0, 1), 2: ((), 3, 1, 2)}

    def __init__(self, rows, static=None):
        self.plan, self.static, self._rows = self._Plan(), static, rows

    def query(self, what, idx):
        assert what == 2
        return [0, self._rows[idx], 0, 0, 0, 0, 0, 0]


def test_last_run_keeps_one_record_per_stream():
    from virconv_b200 import executor

    class Model:
        pass

    m = Model()
    assert executor.last_run(m) is None
    executor.note_last_run(m, _FakeRun({1: 1000, 2: 500}))                  # a one-plan model (VirConvL8x's call)
    executor.note_last_run(m, _FakeRun({1: 3000, 2: 1500}), '_mm')
    executor.note_last_run(m, _FakeRun({1: 1, 2: 1}, static=object()), '_mm')   # a static run's counts stay on the device
    assert executor.last_run(m).rows == {1: 1000, 2: 500}
    assert executor.last_run(m, '_mm').rows == {1: 3000, 2: 1500}
    assert executor.measured_caps(executor.last_run(m, '_mm'), 1.0, 256) == {1: 3072, 2: 1536}
