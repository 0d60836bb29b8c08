"""Static mode promises zero rows past the count in every buffer a step hands on, the slots' input gradients included.  An
arena comes from the caching allocator's pool, so it holds whatever an earlier step or tensor left there: the bf16
static-mode step audit (tests/test_gpu_step_audit.py), run here with every arena filled with a non-zero byte pattern
first, so that no tail can be zero by accident."""
import pytest
import torch

from test_gpu_step_audit import DEV, _audit_l, _batch, _capture, _model

pytestmark = pytest.mark.gpu


def test_static_step_audit_on_dirty_arena(lib_built, monkeypatch):
    from virconv_b200 import executor, ops
    real = executor.empty_scratch

    def dirty(n, dtype, dev):
        t = real(n, dtype, dev)
        if dtype == torch.uint8:     # (the arenas)
            t.fill_(0x3F)
        return t

    monkeypatch.setattr(executor, 'empty_scratch', dirty)
    runs = _capture(monkeypatch)
    model = _model('bf16')
    batch = _batch([0, 1])
    with torch.no_grad():
        model(dict(batch))
    caps = executor.measured_caps(executor.last_run(model), 1.3, 256)
    n = batch['voxel_features'].shape[0]
    cap0 = (int(n * 1.25) + 255) // 256 * 256
    vf = torch.full((cap0, batch['voxel_features'].shape[1]), float('nan'), device=DEV)
    vc = torch.full((cap0, 4), -1.0, device=DEV)
    vf[:n] = batch['voxel_features']
    vc[:n] = batch['voxel_coords']
    spec = executor.StaticSpec(torch.tensor([n], dtype=torch.int32, device=DEV), caps, torch.zeros(1, dtype=torch.int32, device=DEV))
    bd = {'voxel_features': vf, 'voxel_coords': vc, 'batch_size': 2, 'calib': batch['calib'], 'aug_param': batch['aug_param'],
          'virconv_static': spec, 'virconv_proj': ops.projection_params(batch['calib'], batch['aug_param'], 2, DEV)}
    _audit_l(model, bd, runs, 'bf16 static, dirty arenas', static=True)
