"""The deep ResNet constructors' layer counts (reference model/resnet.py:200-224: resnet101 -> Bottleneck [3, 4, 23, 3], resnet152 ->
Bottleneck [3, 8, 36, 3]), registered in the oracle's table of ResNet architectures on import.  Every ResNet restatement is driven by that
table -- `oracle.yolo2_oracle.resnet_blocks / make_resnet_state_dict / resnet_forward`, the train-mode `resnet_train_oracle`, the fp64
teacher of test_train_units.py and tools/resnet_train_error_budget.py -- so importing this module lets all of them run the deep nets with
the same arithmetic that the executed-reference fixtures pin for resnet18 / 50 and, through resnet_deep.npz, for resnet101 / 152."""
from oracle import yolo2_oracle as O

DEEP_LAYERS = {'resnet101': ('bottleneck', (3, 4, 23, 3)), 'resnet152': ('bottleneck', (3, 8, 36, 3))}

for _name, _layers in DEEP_LAYERS.items():
    assert O.RESNET_LAYERS.setdefault(_name, _layers) == _layers, _name
