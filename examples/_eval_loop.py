"""The evaluation demos' batch loop.  By default the host reader feeds EvalUtil batch by batch.  With --device-resident the records
live on the device and DeviceEvalUtil keeps the distances there; with --graph every batch (reading, inference, the script's
post-processing and the feed) is replayed from one CUDA graph (hand3d_b200.train_loop.GraphedIteration), and the host waits once, in
get_measures()."""
from hand3d_b200.train_loop import GraphedIteration
from hand3d_b200.utils.general import DeviceEvalUtil, EvalUtil


def add_flags(ap):
    ap.add_argument("--device-resident", action="store_true",
                    help="upload the records to the GPU once and keep the distances there (DeviceEvalUtil)")
    ap.add_argument("--graph", action="store_true", help="replay each batch from one CUDA graph; needs --device-resident")


def check_flags(ap, args):
    if args.graph and not args.device_resident:
        ap.error("--graph captures the reader too, which needs --device-resident")


def evaluate(dataset, step, n, batch, device_resident=False, graph=False):
    """Runs step(dataset.get(), util) for the ceil(n / batch) batches that cover n samples and returns util.  DeviceEvalUtil keeps the
    first n samples, so a last batch that wraps around the records counts none of them twice."""
    util = DeviceEvalUtil(num_samples=n) if device_resident else EvalUtil()

    def iteration():
        step(dataset.get(), util)

    run = GraphedIteration(iteration) if graph else iteration
    for _ in range(0, n, batch):
        run()
    return util
