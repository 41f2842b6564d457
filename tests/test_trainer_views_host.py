"""CPU-only: the host arithmetic of several views per step -- the symmetric allocation's layout and the rank-major
order of its view pointers (multigpu.symmetric_layout / view_pointers), and the checks a step makes on its cameras
and images before it touches the device (trainer.view_setups)."""
import numpy as np
import pytest
import torch

from opensplat_b200.model import Camera
from opensplat_b200.multigpu import symmetric_layout, view_pointers
from opensplat_b200.parallel import flat_layout
from opensplat_b200.trainer import view_setups


@pytest.mark.parametrize("n", [0, 1, 2, 3, 127, 1001, 4096])
@pytest.mark.parametrize("B", [1, 2, 3, 4, 8, 9])
@pytest.mark.parametrize("G", [1, 2, 3, 8])
def test_symmetric_layout_offsets_alignment_and_rank_major_pointers(n, B, G):
    _, numel = flat_layout(n, 16)
    rgb_off, cam_off, total = symmetric_layout(numel, n, B)
    # [flat gradients | B colour slots | B trailers], nothing overlapping, block and trailers on 16-byte boundaries
    assert rgb_off >= numel and rgb_off % 4 == 0 and rgb_off - numel < 4
    assert cam_off >= rgb_off + 3 * n * B and cam_off % 4 == 0 and cam_off - (rgb_off + 3 * n * B) < 4
    assert total == cam_off + 4 * B
    if B == 1:                                # the single-view layout
        assert (rgb_off, cam_off) == ((numel + 3) // 4 * 4, (numel + 3) // 4 * 4 + (3 * n + 3) // 4 * 4)
    bases = [(1 << 40) + r * (1 << 32) for r in range(G)]     # 16-byte aligned allocations, one per rank
    rgb, cam = view_pointers(bases, n, B, rgb_off, cam_off)
    assert len(rgb) == len(cam) == G * B
    for r in range(G):
        for b in range(B):
            i = r * B + b                      # rank-major: every replica expands the views in the same order
            assert rgb[i] == bases[r] + 4 * rgb_off + 12 * n * b     # slots are contiguous: one mask over n*B
            assert cam[i] == bases[r] + 4 * cam_off + 16 * b and cam[i] % 16 == 0
            assert bases[r] + 4 * numel <= rgb[i] and rgb[i] + 12 * n <= bases[r] + 4 * cam_off
            assert cam[i] + 12 <= bases[r] + 4 * total
    assert len(set(cam)) == G * B and (n == 0 or len(set(rgb)) == G * B)


def test_symmetric_layout_rejects_no_views():
    with pytest.raises(ValueError):
        symmetric_layout(100, 10, 0)


def _cam(W=128, H=96, turn=0.0):
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3, :3] = np.array([[np.cos(turn), 0, -np.sin(turn)], [0, 1, 0], [np.sin(turn), 0, np.cos(turn)]])
    c2w[:3, 3] = [0.0, 0.0, 4.0]
    return Camera(W, H, 0.9 * W, 0.9 * W, W / 2.0, H / 2.0, c2w)


def test_view_setups_takes_b_cameras_and_images():
    cams = [_cam(turn=0.1 * b) for b in range(3)]
    gts = torch.zeros((3, 96, 128, 3))
    setups, H, W = view_setups(cams, gts, 3, 1)
    assert (H, W) == (96, 128) and len(setups) == 3
    assert not torch.equal(setups[0][5], setups[1][5]) or not torch.equal(setups[0][3], setups[1][3])
    setups, H, W = view_setups(cams, list(torch.zeros((3, 48, 64, 3))), 3, 2)     # downscaled, a list of images
    assert (H, W) == (48, 64)


def test_view_setups_rejects_a_wrong_number_of_views():
    cams = [_cam() for _ in range(3)]
    with pytest.raises(ValueError):
        view_setups(cams[:2], torch.zeros((3, 96, 128, 3)), 3, 1)
    with pytest.raises(ValueError):
        view_setups(cams, torch.zeros((2, 96, 128, 3)), 3, 1)
    with pytest.raises(ValueError):
        view_setups(cams[0], torch.zeros((1, 96, 128, 3)), 3, 1)
    with pytest.raises(ValueError):
        view_setups(cams + [_cam()], [torch.zeros((96, 128, 3))] * 4, 3, 1)


def test_view_setups_rejects_mixed_resolutions_and_wrong_images():
    with pytest.raises(ValueError, match="same resolution"):
        view_setups([_cam(), _cam(W=160)], torch.zeros((2, 96, 128, 3)), 2, 1)
    with pytest.raises(ValueError):           # an image at another resolution
        view_setups([_cam(), _cam()], [torch.zeros((96, 128, 3)), torch.zeros((48, 64, 3))], 2, 1)
    with pytest.raises(ValueError):           # not float32
        view_setups([_cam(), _cam()], torch.zeros((2, 96, 128, 3), dtype=torch.float64), 2, 1)
