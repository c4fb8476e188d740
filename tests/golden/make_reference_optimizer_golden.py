"""Pins the parameter order and the optimizer-state format of a reference checkpoint — by running the reference's own module
under ``torch.optim.Adam``.

A reference run is resumed from a Lightning checkpoint whose ``optimizer_states[0]`` is ``torch.optim.Adam.state_dict()`` of
``FlowGNNGGNNModule.parameters()`` (config_default.yaml:43-47: lr 1e-3, weight_decay 1e-2).  Its parameter indices follow the
reference module's ``named_parameters()`` order, which is what ``FusedTrainer.optimizer.load_state_dict`` has to map onto
its flat buffers.  This script builds the REAL reference class (same stand-ins as make_reference_ctrlflow_golden.py: the
bookkeeping packages, and the two DGL operators bound to the oracle restatements), takes a few Adam steps on seeded synthetic
batches and stores:

    names        the reference's named_parameters() order
    state_dict   the module's parameters after those steps
    optimizer    opt.state_dict() at that point (what optimizer_states[0] holds)
    next_graph   the next batch
    loss_next / state_after   the training loss on it and the parameters after one more reference Adam step

Run with a checkout of the reference project:   python tests/golden/make_reference_optimizer_golden.py <reference root>
Writes tests/golden/reference_optimizer_golden.pt, read by tests/test_optimizer_state.py and tests/test_trainer_state_gpu.py.
"""
import copy
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from deepdfa_b200 import synth  # noqa: E402
from make_reference_ctrlflow_golden import install_stand_ins  # noqa: E402

CTOR = dict(feat="_ABS_DATAFLOW_datatype_all_limitall_1000_limitsubkeys_1000", input_dim=32, hidden_dim=4, n_steps=3,
            num_output_layers=2, concat_all_absdf=True)
LR, WEIGHT_DECAY, STEPS = 1e-3, 1e-2, 3


def graph_record(g):
    src, dst = g.edges()
    return {"src": src, "dst": dst, "batch_num_nodes": g.batch_num_nodes(), "ndata": dict(g.ndata)}


def main(reference_root):
    install_stand_ins()
    sys.path.insert(0, os.path.join(reference_root, "DDFA"))
    from code_gnn.models.flow_gnn.ggnn import FlowGNNGGNNModule as RefModule      # the real reference class

    torch.manual_seed(31)
    ref = RefModule(**CTOR)
    ref.train()
    opt = torch.optim.Adam(ref.parameters(), lr=LR, weight_decay=WEIGHT_DECAY)
    batches = [synth.make_batch(sizes=[9, 14, 3, 20, 6], seed=40 + i, vuln_rate=0.4, input_dim=CTOR["input_dim"])
               for i in range(STEPS + 1)]
    losses = []
    for g in batches[:STEPS]:
        opt.zero_grad()
        loss = ref.training_step((g, {}), 0)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    fixture = {"ctor": CTOR, "lr": LR, "weight_decay": WEIGHT_DECAY, "losses": losses,
               "names": [n for n, _ in ref.named_parameters()],
               "state_dict": {k: v.clone() for k, v in ref.state_dict().items()},
               "optimizer": copy.deepcopy(opt.state_dict()),
               "next_graph": graph_record(batches[STEPS])}
    opt.zero_grad()
    loss = ref.training_step((batches[STEPS], {}), 0)
    loss.backward()
    opt.step()
    fixture["loss_next"] = float(loss.detach())
    fixture["state_after"] = {k: v.clone() for k, v in ref.state_dict().items()}
    fixture["note"] = "reference ggnn.py / base_module.py under torch.optim.Adam; DGL ops bound to the oracle restatements"
    out = os.path.join(ROOT, "tests", "golden", "reference_optimizer_golden.pt")
    torch.save(fixture, out)
    print("wrote", out, f"{os.path.getsize(out)} bytes,", len(fixture["names"]), "parameters, losses", losses, fixture["loss_next"])


if __name__ == "__main__":
    main(sys.argv[1])
