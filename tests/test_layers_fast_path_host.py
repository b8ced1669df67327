"""CPU tests of which geometries the staged bias+ReLU+max-pool kernels take (cos_pool_fast_path, a pure host function)
and of the process-wide switch that forces the reference kernels.  No device compute is attempted here."""
import pytest

# (N, C, H, W) of the bias-free conv output, pool kernel, stride
FAST = {
    "caffenet_conv1_b256": (256, 96, 55, 55, 3, 2),
    "caffenet_conv2_b256": (256, 256, 27, 27, 3, 2),
    "caffenet_conv5_b256": (256, 256, 13, 13, 3, 2),
    "caffenet_conv1_b1": (1, 96, 55, 55, 3, 2),
    "cifar10_quick_conv1_b100": (100, 32, 32, 32, 3, 2),
    "cifar10_quick_conv1_b1": (1, 32, 32, 32, 3, 2),
    "k2s2": (64, 20, 24, 24, 2, 2),
    "k3s1": (2, 3, 9, 10, 3, 1),
    "k5s3": (2, 3, 13, 12, 5, 3),
    "h_equals_k": (2, 3, 3, 3, 3, 2),
    "plane_near_smem_limit": (2, 2, 90, 100, 3, 2),  # the backward stages 47,338 bytes per plane
}
FALLBACK = {
    "x_plane_past_48k": (2, 2, 111, 111, 3, 2),  # 49,284 bytes of fp32 x
    "bwd_plane_past_48k": (2, 2, 100, 120, 3, 2),  # x fits (48,064 bytes); g, dy and index do not (63,080)
    "large_plane": (1, 1, 1024, 1024, 3, 2),
    "k1s1": (2, 3, 5, 6, 1, 1),
    "k1s2": (2, 3, 7, 6, 1, 2),
    "k4s1": (2, 3, 9, 9, 4, 1),  # k > s + 2
    "k7s2": (2, 3, 15, 16, 7, 2),
    "k15s1": (1, 2, 17, 16, 15, 1),
    "h_below_k": (2, 3, 2, 9, 3, 2),
    "w_below_k": (2, 3, 9, 2, 3, 2),
    "plane_1x1": (2, 3, 1, 1, 3, 2),
    "plane_1x1_k1": (2, 3, 1, 1, 1, 1),
    "empty_batch": (0, 3, 9, 9, 3, 2),
    "no_channels": (2, 0, 9, 9, 3, 2),
    "stride_0": (2, 3, 9, 9, 3, 0),
    "outputs_past_2g": (65536, 512, 129, 129, 3, 2),  # 2^25 planes x 64^2 outputs: past 32-bit indices
}


@pytest.mark.parametrize("case", list(FAST))
def test_net_geometries_take_the_staged_kernels(cos, case):
    from caffeonspark_b200 import _lib
    assert _lib.lib().cos_pool_fast_path(*FAST[case]) == 1


@pytest.mark.parametrize("case", list(FALLBACK))
def test_other_geometries_take_the_reference_kernels(cos, case):
    from caffeonspark_b200 import _lib
    assert _lib.lib().cos_pool_fast_path(*FALLBACK[case]) == 0


def test_fast_path_does_not_depend_on_the_switch(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    was = L.cos_layers_reference_kernels()
    try:
        for on in (1, 0):
            L.cos_layers_set_reference_kernels(on)
            assert L.cos_layers_reference_kernels() == on
            assert L.cos_pool_fast_path(*FAST["caffenet_conv1_b256"]) == 1
    finally:
        L.cos_layers_set_reference_kernels(was)


@pytest.mark.parametrize("value,want", [(None, 0), ("0", 0), ("", 0), ("1", 1)])
def test_switch_starts_from_the_environment(cos, value, want):
    # the variable is read once when the library loads: load it in a fresh interpreter
    import os
    import subprocess
    import sys
    env = dict(os.environ)
    env.pop("COS_LAYERS_REFERENCE_KERNELS", None)
    if value is not None:
        env["COS_LAYERS_REFERENCE_KERNELS"] = value
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "from caffeonspark_b200 import _lib; print(_lib.lib().cos_layers_reference_kernels())"
    out = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, check=True)
    assert out.stdout.strip() == str(want)
