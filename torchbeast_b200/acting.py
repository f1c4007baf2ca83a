"""The T=1 acting forward replayed as a CUDA graph (GraphedActor).

An inference thread (polybeast_learner.inference, reference polybeast_learner.py:269-285) or monobeast's act() runs the
acting forward once per environment step, for B = 1 .. 512 actors.  Eagerly, every call pays the host launch cost of
every kernel of the network; a replay pays one graph launch plus the copies into the graph's static inputs.

    actor = GraphedActor(model)
    outputs, core_state = actor(inputs, core_state)   # exactly what model(inputs, core_state) returns

* One graph per (bucket, model.training, model.precision, input dtypes): the bucket is the next power of two >= B.
  Every kernel-selection threshold on B in the network is 32, so padding a call to its bucket never moves it to another
  kernel.  The real rows are copied into columns [:B] of the graph's static inputs and the outputs are returned sliced
  to [:B]; padded rows never reach the caller.
* Each graph owns every buffer it reads or writes: its static inputs and outputs, the model workspace it was captured
  with (the model's cached workspace is replaced when another shape is run) and its device (seed, step) pair.
* Training mode samples with the model's `action_sampler` (torchbeast_b200.sampling.ActionSampler), which is required.
  The captured sampler launch reads (seed, step) from device memory (tb_sample_actions_dev_f32); before each replay the
  seed and step of the sampler attached at that moment are published there, and the sampler's step then advances by one
  on the host, as an eager call advances it.  Graphed and eager calls can therefore be mixed freely.  Eval mode is greedy.
* The weights are read from the model's flat parameter buffer inside the graph, so copy_params_from / load_state_dict
  show up in the next replay.  If the buffer moves (.to(), .cuda()), the graphs are dropped and captured again.
* Outputs are views of the graph's static buffers, valid until the next call on the same GraphedActor; calls must be
  serialised by the caller (polybeast_learner.inference holds its lock around the call).
"""
import torch

from torchbeast_b200 import _lib


def bucket_size(B):
    """The batch size a call of B rows is padded to: the next power of two >= B."""
    if B < 1:
        raise _lib.TorchBeastB200Error("batch size must be at least 1, got %d" % B)
    return 1 << (B - 1).bit_length()


def _as_int64(x):
    """An unsigned 64-bit value (taken mod 2^64) as the int64 with the same bits."""
    x %= 2 ** 64
    return x - 2 ** 64 if x >= 2 ** 63 else x


def replay_sampler(model):
    """The sampler a replay publishes (seed, step) from: model.action_sampler in training mode, where it is required
    (torch.multinomial cannot be replayed at a new step), and None in eval mode, which is greedy."""
    if not model.training:
        return None
    if model.action_sampler is None:
        raise _lib.TorchBeastB200Error(
            "GraphedActor in training mode needs model.action_sampler (torchbeast_b200.sampling.ActionSampler)")
    return model.action_sampler


def _rows(nest, B):
    """Columns [:B] of every [T or layers, bucket, ...] leaf."""
    if isinstance(nest, torch.Tensor):
        return nest[:, :B]
    if isinstance(nest, dict):
        return {k: _rows(v, B) for k, v in nest.items()}
    return tuple(_rows(v, B) for v in nest)


class _DeviceStepSampler:
    """Stands in for model.action_sampler while a graph is warmed up and captured: its launch reads (seed, step) from
    `seed_step` (int64 [2] on the device) when it runs, so the user's sampler is neither read nor advanced here."""

    def __init__(self, seed_step):
        self.seed_step = seed_step

    def sample(self, logits, stream_ids=None):
        T, B, A = logits.shape
        logits = logits.detach().contiguous()
        if stream_ids is not None:
            stream_ids = stream_ids.to(device=logits.device, dtype=torch.int64).contiguous()
        actions = torch.empty(T, B, dtype=torch.int64, device=logits.device)
        _lib.check(
            _lib.lib().tb_sample_actions_dev_f32(_lib.ptr(logits), T, B, A, _lib.ptr(self.seed_step),
                                                 _lib.ptr(stream_ids), _lib.ptr(actions), _lib.stream_ptr()),
            "tb_sample_actions_dev_f32")
        return actions


class _Graph:
    """One captured acting forward and every buffer it uses."""

    def __init__(self, graph, inputs, state, seed_step, workspace, outputs, new_state):
        self.graph, self.inputs, self.state, self.seed_step = graph, inputs, state, seed_step
        self.workspace = workspace  # keeps the captured workspace alive when the model replaces its own
        self.outputs, self.new_state = outputs, new_state
        self.default_ids = True     # inputs["stream_ids"] holds the column indices (the default stream ids)


class GraphedActor:
    """model(inputs, core_state) for T = 1 as a CUDA-graph replay; see the module docstring."""

    WARMUP_CALLS = 2

    def __init__(self, model):
        if not model.flat_params.is_cuda:
            raise _lib.TorchBeastB200Error("GraphedActor needs a model on a CUDA device, got %s" % model.flat_params.device)
        self.model = model
        self._graphs = {}
        self._flat_ptr = model.flat_params.data_ptr()
        self.captures = 0  # graphs captured so far (a recapture after the weights moved counts again)

    def _input_names(self):
        return ("frame", "reward", "done", "last_action") if getattr(self.model, "needs_last_action", False) \
            else ("frame", "reward", "done")

    def __call__(self, inputs, core_state=()):
        model = self.model
        if inputs["frame"].dim() != 5:
            raise _lib.TorchBeastB200Error("GraphedActor takes stacked frames [1, B, 4, 84, 84]; unstacked rollouts are a "
                                           "learner input, got frame %r" % (tuple(inputs["frame"].shape),))
        sampler = replay_sampler(model)
        _lib.require_cuda(model.flat_params)
        T, B = inputs["frame"].shape[:2]
        if T != 1:
            raise _lib.TorchBeastB200Error("GraphedActor replays the T=1 acting forward, got T=%d" % T)
        if model.flat_params.data_ptr() != self._flat_ptr:  # the weights moved: every graph reads the old address
            self._graphs.clear()
            self._flat_ptr = model.flat_params.data_ptr()
        names = self._input_names()
        key = (bucket_size(B), model.training, model.precision, tuple(inputs[k].dtype for k in names))
        with torch.no_grad():
            g = self._graphs.get(key)
            if g is None:
                g = self._graphs[key] = self._capture(key[0], inputs, names)
            if len(core_state) != len(g.state):
                raise _lib.TorchBeastB200Error("core_state has %d tensors, the model's has %d" % (len(core_state), len(g.state)))
            for k in names:
                g.inputs[k][:, :B].copy_(inputs[k], non_blocking=True)
            for dst, src in zip(g.state, core_state):
                dst[:, :B].copy_(src, non_blocking=True)
            if sampler is not None:
                ids = inputs.get("stream_ids")
                if ids is not None:
                    g.inputs["stream_ids"][:B].copy_(ids, non_blocking=True)
                    g.default_ids = False
                elif not g.default_ids:
                    g.inputs["stream_ids"].copy_(torch.arange(key[0], dtype=torch.int64), non_blocking=True)
                    g.default_ids = True
                # a fresh pinned block: the caching host allocator does not hand it out again until this copy is done
                host = torch.empty(2, dtype=torch.int64, pin_memory=True)
                host.numpy()[:] = (_as_int64(sampler.seed), _as_int64(sampler.step))
                g.seed_step.copy_(host, non_blocking=True)
            g.graph.replay()
            if sampler is not None:
                sampler.step += T
        return _rows(g.outputs, B), _rows(g.new_state, B)

    def _capture(self, Bk, inputs, names):
        model = self.model
        dev = model.flat_params.device
        static = {k: torch.zeros((1, Bk) + tuple(inputs[k].shape[2:]), dtype=inputs[k].dtype, device=dev) for k in names}
        if model.training:
            static["stream_ids"] = torch.arange(Bk, dtype=torch.int64, device=dev)
        state = tuple(model.initial_state(Bk))
        seed_step = torch.zeros(2, dtype=torch.int64, device=dev)
        saved = model.action_sampler
        model.action_sampler = _DeviceStepSampler(seed_step)
        try:
            # warm up on a side stream (workspace, LSTM side stream, module loads), then capture
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(self.WARMUP_CALLS):
                    model(static, state)
            torch.cuda.current_stream(dev).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            # thread-local: another thread (a learner) may allocate or synchronise while this one captures
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                outputs, new_state = model(static, state)
        finally:
            model.action_sampler = saved
        self.captures += 1
        return _Graph(graph, static, state, seed_step, getattr(model, "_ws", None), outputs, tuple(new_state))
