"""etxb_destroy / etxb_group_destroy free every device buffer a context or a group allocated: cycles of create, upload, render one iteration
and destroy leave the device's free memory where they found it.  The scene is a stochastic-BSDF box (connection, sort and shadow-list
buffers, the 4-wide tree) at a film whose light-vertex pool alone is about 200 MB, so one leaked context shows far above the slack."""
import pytest

from etx_tracer_b200 import scenes

gpu = pytest.mark.gpu
CYCLES = 5
SLACK = 16 << 20  # allocator granularity and the runtime's own bookkeeping


def _scene():
    return scenes.material_box("plastic", 256, 256, samples=16)


def _free_after_cycles(make, scene):
    import torch
    levels = []
    for _ in range(CYCLES + 1):  # the first cycle loads the module and creates the device's context: the level is taken after it
        g = make(scene)
        g.render(1)
        g.close()
        torch.cuda.synchronize()
        levels.append(torch.cuda.mem_get_info()[0])
    return levels


@gpu
@pytest.mark.parametrize("integrator", ["vcm", "pt"])
def test_context_destroy_frees_device_memory(integrator):
    from etx_tracer_b200 import api
    cls = api.GPUVCM if integrator == "vcm" else api.GPUPathTracing
    levels = _free_after_cycles(lambda sd: cls(sd, flavor="fast"), _scene())
    assert abs(levels[-1] - levels[0]) <= SLACK, [f"{(x - levels[0]) / 2**20:.1f} MB" for x in levels]


@gpu
def test_group_destroy_frees_device_memory():
    from etx_tracer_b200 import api
    levels = _free_after_cycles(lambda sd: api.GPUVCMGroup(sd, lanes=2, flavor="fast"), _scene())
    assert abs(levels[-1] - levels[0]) <= SLACK, [f"{(x - levels[0]) / 2**20:.1f} MB" for x in levels]
