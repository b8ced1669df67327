"""CPU tests of the layout parser's refusals, each with its exact wording and the layer it names, and of Deconvolution:
its weight shape C_in x (num_output / group) x kh x kw, its bias and its output shape."""
import pytest

# a 2x3x4x5 Input `x` and its 2 labels
INPUT = ('layer { name: "in" type: "Input" top: "x" top: "label" input_param { shape { dim: 2 dim: 3 dim: 4 dim: 5 } '
         'shape { dim: 2 } } }\n')


def _solver(tmp_path, net):
    (tmp_path / "net.prototxt").write_text('name: "t"\n' + net)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    return str(tmp_path / "solver.prototxt")


@pytest.mark.parametrize("net,message", [
    (INPUT + 'layer { name: "r" type: "ReLU" bottom: "nope" top: "y" }', "layer 'r' (ReLU): unknown bottom blob"),
    (INPUT + 'layer { name: "r" type: "ReLU" top: "y" }', "layer 'r' (ReLU): unknown bottom blob"),
    # an unknown bottom is reported before the convolution's own check
    (INPUT + 'layer { name: "c" type: "Convolution" bottom: "nope" top: "y" convolution_param { num_output: 4 '
     'kernel_size: 3 } }', "layer 'c' (Convolution): unknown bottom blob"),
    (INPUT + 'layer { name: "c" type: "Convolution" bottom: "label" top: "y" convolution_param { num_output: 4 '
     'kernel_size: 3 } }', "layer 'c': bad Convolution"),
    (INPUT + 'layer { name: "c" type: "Convolution" bottom: "x" top: "y" }', "layer 'c': bad Convolution"),
    (INPUT + 'layer { name: "c" type: "Convolution" bottom: "x" top: "y" convolution_param { num_output: 4 } }',
     "layer 'c': bad convolution_param"),
    (INPUT + 'layer { name: "c" type: "Convolution" bottom: "x" top: "y" convolution_param { num_output: 4 '
     'kernel_size: 3 group: 2 } }', "layer 'c': bad convolution_param"),
    (INPUT + 'layer { name: "p" type: "Pooling" bottom: "x" top: "y" }', "layer 'p': bad Pooling"),
    (INPUT + 'layer { name: "p" type: "Pooling" bottom: "x" top: "y" pooling_param { pool: MAX } }',
     "layer 'p': bad pooling_param"),
    (INPUT + 'layer { name: "ip" type: "InnerProduct" bottom: "x" top: "y" }', "layer 'ip': bad InnerProduct"),
    (INPUT + 'layer { name: "ip" type: "InnerProduct" bottom: "x" top: "y" inner_product_param { num_output: 0 } }',
     "layer 'ip': bad inner_product_param"),
    (INPUT + 'layer { name: "ip" type: "InnerProduct" bottom: "x" top: "y" inner_product_param { num_output: 3 '
     'axis: 5 } }', "layer 'ip': bad inner_product_param"),
    ('layer { name: "d" type: "MemoryData" top: "x" top: "label" }', "MemoryData layer without memory_data_param"),
    ('layer { name: "d" type: "CoSData" top: "x" top: "label" }', "CoSData layer without cos_data_param"),
    # an Input top with no shape has no axes
    ('layer { name: "z" type: "Input" top: "z" }\nlayer { name: "bn" type: "BatchNorm" bottom: "z" top: "z" }',
     "layer 'bn': bad BatchNorm bottom"),
    ('layers { name: "r" type: RELU bottom: "x" top: "x" }', "V1 'layers' net definitions are not supported"),
    (INPUT + 'layer { name: "sl" type: "Slice" bottom: "x" }', "layer 'sl' (Slice): needs at least one top"),
    ('layer { name: "z" type: "Input" top: "z" }\nlayer { name: "f" type: "Flatten" bottom: "z" top: "y" }',
     "layer 'f' (Flatten): axis 1 out of range for 0-D Blob"),
])
def test_refusal_wording(cos, tmp_path, net, message):
    with pytest.raises(cos.CosError) as e:
        cos.parse_solver(_solver(tmp_path, net))
    assert str(e.value) == message


@pytest.mark.parametrize("group,weight", [(1, 3 * 6 * 3 * 3), (3, 3 * 2 * 3 * 3)])
def test_deconvolution_counts(cos, tmp_path, group, weight):
    # the weight count equals Convolution's, so this pins the bias and the output shape:
    # out H = 2 * (4 - 1) + 3 - 2 * 1 = 7 and W = 2 * (5 - 1) + 3 - 2 = 9, read back through the InnerProduct's weight
    net = (INPUT + f'layer {{ name: "d" type: "Deconvolution" bottom: "x" top: "y" convolution_param {{ num_output: 6 '
           f'kernel_size: 3 stride: 2 pad: 1 group: {group} }} }}\n'
           'layer { name: "ip" type: "InnerProduct" bottom: "y" top: "ip" inner_product_param { num_output: 3 } }\n'
           'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')
    assert cos.parse_solver(_solver(tmp_path, net)).counts == [weight, 6, 3 * 6 * 7 * 9, 3]
    net = net.replace("kernel_size: 3", "kernel_size: 3 bias_term: false")
    assert cos.parse_solver(_solver(tmp_path, net)).counts == [weight, 3 * 6 * 7 * 9, 3]


@pytest.mark.parametrize("group,deconv,conv", [(1, "3 6 3 3 (162)", "6 3 3 3 (162)"), (3, "3 2 3 3 (54)", "6 1 3 3 (54)")])
def test_deconvolution_weight_shape(cos, tmp_path, group, deconv, conv):
    # A Convolution with the same count cannot share the Deconvolution's weight: the refusal names both blob shapes.
    param = f'convolution_param {{ num_output: 6 kernel_size: 3 group: {group} }} param {{ name: "w" }}'
    net = (INPUT + f'layer {{ name: "d" type: "Deconvolution" bottom: "x" top: "y" {param} }}\n'
           f'layer {{ name: "c" type: "Convolution" bottom: "x" top: "z" {param} }}\n')
    with pytest.raises(cos.CosError) as e:
        cos.parse_solver(_solver(tmp_path, net))
    assert str(e.value) == (f"Cannot share param 'w' owned by layer 'd' with layer 'c'; shape mismatch.  Owner layer "
                            f"param shape is {deconv}; sharing layer expects shape {conv}")
