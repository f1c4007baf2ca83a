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
* With inputs["legal_actions"] (bool or uint8 [1, B, A], torchbeast_b200.legal_actions) the mask is one more static
  input, and its presence is part of the graph key: the forward masks its logits, so the sampled and greedy actions
  are legal.  Padding columns hold an all-zero row, which leaves their logits unmasked.
* With a FrameHistory attached as `model.frame_history`, a call may pass each stream's newest frame u8 [1, B, 84, 84]
  instead of its stack, with inputs["stream_ids"] naming the streams (default: the column indices).  The graph's static
  frame is then the unstacked array [4, Bk, 84, 84]: the call's frames go to row 3 and the captured history fill writes
  rows 0..2.  Padding columns get stream id -1 and leave every history alone.  Such graphs are keyed by the history's
  buffer and size, and hold that buffer and (on the backends that restack) the model's stacked scratch they were
  captured with.  Eager calls and replays on one history must
  be serialised like any two calls here.
"""
import torch

from torchbeast_b200 import _lib, nets, sampling


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


class FrameHistory:
    """The last three frames of each of `num_streams` actor streams, on the device, so an acting call can send each
    stream's newest frame u8 [1, B, 84, 84] and have its four-frame stack rebuilt there.

        model.frame_history = FrameHistory(num_envs)
        outputs, core_state = model(dict(inputs, frame=newest, stream_ids=env_ids), core_state)

    `buffer` (u8 [S, 3, 84, 84]) holds, oldest first, channels 1..3 of the stack each stream's last call used; a new
    history is all zeros.  inputs["stream_ids"] (int64 [B]; default: the column indices) picks each column's stream,
    as it picks the sampler's random stream, and the ids of one call must be distinct.  The buffer never moves, because
    captured graphs read it by address.  Calls that share a history must be serialised, by one lock or one CUDA stream
    (include/torchbeast_b200.h, tb_frame_history_fill_u8)."""

    def __init__(self, num_streams, device=None):
        if int(num_streams) < 1:
            raise _lib.TorchBeastB200Error("FrameHistory needs num_streams >= 1, got %r" % (num_streams,))
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.buffer = torch.zeros(int(num_streams), 3, 84, 84, dtype=torch.uint8, device=device)

    @property
    def num_streams(self):
        return self.buffer.shape[0]

    @property
    def device(self):
        return self.buffer.device

    def reset(self, stream_ids=None):
        """Zero every stream's history, or those of `stream_ids`."""
        if stream_ids is None:
            self.buffer.zero_()
        else:
            ids = torch.as_tensor(stream_ids, dtype=torch.int64).to(self.buffer.device)
            self.buffer.index_fill_(0, ids, 0)

    def fill(self, frames, done, stream_ids):
        """Rows 0..2 of the unstacked array frames u8 [T+3, B, 84, 84] (rows 3.. already hold the newest frames) from
        the history at stream_ids (int64 [B] on the device; an id outside [0, S) gives zero rows and touches no
        history), then each stream's history advanced past step T-1.  done: [T, B] bool or uint8.  Every tensor must
        be contiguous and on the history's device: the kernel takes them as raw pointers."""
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[0] < 4 or tuple(frames.shape[2:]) != (84, 84) \
                or not frames.is_contiguous():
            raise _lib.TorchBeastB200Error("fill: frames must be contiguous uint8 [T+3, B, 84, 84] with T >= 1, got %s %r"
                                           % (frames.dtype, tuple(frames.shape)))
        T, B = frames.shape[0] - 3, frames.shape[1]
        if done.dtype not in (torch.bool, torch.uint8) or tuple(done.shape) != (T, B) or not done.is_contiguous():
            raise _lib.TorchBeastB200Error("fill: done must be contiguous bool or uint8 [%d, %d], got %s %r"
                                           % (T, B, done.dtype, tuple(done.shape)))
        if stream_ids.dtype != torch.int64 or tuple(stream_ids.shape) != (B,) or not stream_ids.is_contiguous():
            raise _lib.TorchBeastB200Error("fill: stream_ids must be contiguous int64 [%d], got %s %r"
                                           % (B, stream_ids.dtype, tuple(stream_ids.shape)))
        if any(t.device != self.device for t in (frames, done, stream_ids)):
            raise _lib.TorchBeastB200Error("fill: frames, done and stream_ids must be on the history's device %s, got %s"
                                           % (self.device, [str(t.device) for t in (frames, done, stream_ids)]))
        _lib.require_cuda(self.buffer)
        _lib.check(
            _lib.lib().tb_frame_history_fill_u8(_lib.ptr(frames), _lib.ptr(done), _lib.ptr(stream_ids), T, B, 84 * 84,
                                                _lib.ptr(self.buffer), self.num_streams, _lib.stream_ptr()),
            "tb_frame_history_fill_u8")

    def stack(self, frame, done, stream_ids, device):
        """The unstacked array [T+3, B, 84, 84] for newest frames frame u8 [T, B, 84, 84] with done [T, B] (bool or
        uint8), rows 0..2 filled from this history (see fill).  CPU stream_ids are checked here: distinct and in
        [0, num_streams); ids already on the device are trusted."""
        if frame.dtype != torch.uint8 or frame.dim() != 4 or tuple(frame.shape[2:]) != (84, 84):
            raise _lib.TorchBeastB200Error("with a frame_history, frame must be the newest frames uint8 [T, B, 84, 84] "
                                           "or an unstacked rollout [T+3, B, 84, 84], got %s %r"
                                           % (frame.dtype, tuple(frame.shape)))
        T, B = frame.shape[:2]
        if device != self.device:
            raise _lib.TorchBeastB200Error("the frame_history is on %s, the model on %s" % (self.device, device))
        done = nets._done_bytes(done, T, B)
        stream_ids = self.checked_ids(stream_ids, B)
        if stream_ids is None:
            stream_ids = torch.arange(B, dtype=torch.int64, device=device)
        else:
            stream_ids = stream_ids.to(device=device, dtype=torch.int64).contiguous()
        _lib.require_cuda(frame, done)
        frames = torch.empty((T + 3, B, 84, 84), dtype=torch.uint8, device=device)
        frames[3:].copy_(frame)
        self.fill(frames, done, stream_ids)
        return frames

    def checked_ids(self, stream_ids, B):
        """stream_ids, after checking it is an integer [B] tensor and, on the host, that its ids are distinct and in
        [0, num_streams).  Ids already on the device are not read back.  None (the column indices) needs B <= S."""
        if stream_ids is None:
            if B > self.num_streams:
                raise _lib.TorchBeastB200Error("the default stream ids 0..%d need a FrameHistory of at least %d streams, "
                                               "this one has %d" % (B - 1, B, self.num_streams))
            return None
        if tuple(stream_ids.shape) != (B,) or stream_ids.dtype.is_floating_point or stream_ids.dtype == torch.bool:
            raise _lib.TorchBeastB200Error("stream_ids must be integer [B] = [%d], got %s %r"
                                           % (B, stream_ids.dtype, tuple(stream_ids.shape)))
        if not stream_ids.is_cuda:
            ids = stream_ids.tolist()
            if len(set(ids)) != len(ids) or any(i < 0 or i >= self.num_streams for i in ids):
                raise _lib.TorchBeastB200Error("stream_ids must be distinct and in [0, %d), got %r" % (self.num_streams, ids))
        return stream_ids


class _DeviceStepSampler:
    """Stands in for model.action_sampler while a graph is warmed up and captured: its launch reads (seed, step) from
    `seed_step` (int64 [2] on the device) when it runs, so the user's sampler is neither read nor advanced here."""

    def __init__(self, seed_step):
        self.seed_step = seed_step

    def sample(self, logits, stream_ids=None, action_dims=None, continuous_dim=None):
        T, B, A = logits.shape
        logits = logits.detach().contiguous()
        if stream_ids is not None:
            stream_ids = stream_ids.to(device=logits.device, dtype=torch.int64).contiguous()
        if action_dims is not None:  # a factored policy: one entry reads seed_step the same way
            return sampling.sample_factored(logits, action_dims, stream_ids, seed_step=self.seed_step)
        if continuous_dim is not None:  # a Gaussian policy: likewise
            return sampling.sample_gaussian(logits, continuous_dim, stream_ids, seed_step=self.seed_step)
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

    def _input_names(self, inputs):
        names = ("frame", "reward", "done", "last_action") if getattr(self.model, "needs_last_action", False) \
            else ("frame", "reward", "done")
        return names + (("legal_actions",) if inputs.get("legal_actions") is not None else ())

    def __call__(self, inputs, core_state=()):
        model = self.model
        frame, history = inputs["frame"], model.frame_history
        obs = tuple(getattr(model, "observation_shape", nets.ATARI_SHAPE))
        newest = history is not None and frame.dim() == 4
        if (frame.dim() != 5 and not newest) or (frame.dim() == 5 and tuple(frame.shape[2:]) != obs):
            raise _lib.TorchBeastB200Error("GraphedActor takes stacked frames [1, B, %d, %d, %d]; unstacked rollouts are a "
                                           "learner input, got frame %r" % (obs + (tuple(inputs["frame"].shape),)))
        if history is not None and obs != nets.ATARI_SHAPE:
            raise _lib.TorchBeastB200Error("a frame_history rebuilds (4, 84, 84) stacks; this net takes stacked frames "
                                           "[1, B, %d, %d, %d]: detach the history (model.frame_history = None)" % obs)
        channels = tuple(getattr(model, "channels", nets.RESNET_CHANNELS))
        if history is not None and channels != nets.RESNET_CHANNELS:
            raise _lib.TorchBeastB200Error("a frame_history feeds the default widths %r; this net has channels=%r and "
                                           "takes stacked frames: detach the history (model.frame_history = None)"
                                           % (nets.RESNET_CHANNELS, channels))
        if newest and (frame.dtype != torch.uint8 or tuple(frame.shape[2:]) != (84, 84)):
            raise _lib.TorchBeastB200Error("GraphedActor with a frame_history takes stacked frames or the newest frames "
                                           "uint8 [1, B, 84, 84], got %s %r" % (frame.dtype, tuple(frame.shape)))
        sampler = replay_sampler(model)
        _lib.require_cuda(model.flat_params)
        T, B = frame.shape[:2]
        if T != 1:
            raise _lib.TorchBeastB200Error("GraphedActor replays the T=1 acting forward, got T=%d" % T)
        if model.flat_params.data_ptr() != self._flat_ptr:  # the weights moved: every graph reads the old address
            self._graphs.clear()
            self._flat_ptr = model.flat_params.data_ptr()
        names = self._input_names(inputs)
        key = (bucket_size(B), model.training, model.precision, tuple((k, inputs[k].dtype) for k in names),
               "newest" if newest else "stacked",
               (history.buffer.data_ptr(), history.num_streams) if newest else None)
        ids = inputs.get("stream_ids")
        if newest:
            if history.device != model.flat_params.device:
                raise _lib.TorchBeastB200Error("the frame_history is on %s, the model on %s"
                                               % (history.device, model.flat_params.device))
            ids = history.checked_ids(ids, B)
        with torch.no_grad():
            g = self._graphs.get(key)
            if g is None:
                g = self._graphs[key] = self._capture(key[0], inputs, names, history if newest else None)
            if len(core_state) != len(g.state):
                raise _lib.TorchBeastB200Error("core_state has %d tensors, the model's has %d" % (len(core_state), len(g.state)))
            for k in names:
                dst = g.inputs[k][3:] if newest and k == "frame" else g.inputs[k]  # newest frames go to row 3
                dst[:, :B].copy_(inputs[k], non_blocking=True)
            for dst, src in zip(g.state, core_state):
                dst[:, :B].copy_(src, non_blocking=True)
            if newest:  # the history and the sampler read the same ids
                self._set_history_ids(g, ids, B)
            elif sampler is not None:
                if ids is not None:
                    g.inputs["stream_ids"][:B].copy_(ids, non_blocking=True)
                    g.default_ids = False
                elif not g.default_ids:
                    g.inputs["stream_ids"].copy_(torch.arange(key[0], dtype=torch.int64), non_blocking=True)
                    g.default_ids = True
            if sampler is not None:
                # a fresh pinned block: the caching host allocator does not hand it out again until this copy is done
                host = torch.empty(2, dtype=torch.int64, pin_memory=True)
                host.numpy()[:] = (_as_int64(sampler.seed), _as_int64(sampler.step))
                g.seed_step.copy_(host, non_blocking=True)
            g.graph.replay()
            if sampler is not None:
                sampler.step += T
        return _rows(g.outputs, B), _rows(g.new_state, B)

    @staticmethod
    def _set_history_ids(g, ids, B):
        """Columns [:B] of a newest-frame graph's stream ids := ids (default: the column indices).  Every other column
        is -1, so a padding column neither reads nor writes any stream's history."""
        sid = g.inputs["stream_ids"]
        if ids is not None:
            sid[:B].copy_(ids, non_blocking=True)
            g.default_ids = False
        elif not (g.default_ids and g.real_rows >= B):
            sid[:B].copy_(torch.arange(B, dtype=torch.int64), non_blocking=True)
            g.default_ids = True
        if g.real_rows > B:
            sid[B:g.real_rows].fill_(-1)
        g.real_rows = B

    def _capture(self, Bk, inputs, names, history=None):
        """With a history, the static frame is the unstacked array [4, Bk, 84, 84] (calls write row 3) and the graph
        runs the history fill before the forward."""
        model = self.model
        dev = model.flat_params.device
        static = {k: torch.zeros((1, Bk) + tuple(inputs[k].shape[2:]), dtype=inputs[k].dtype, device=dev) for k in names}
        if history is not None:
            static["frame"] = torch.zeros(4, Bk, 84, 84, dtype=torch.uint8, device=dev)
            # -1 until a call writes its ids: the warm-up fills neither read nor write the history
            static["stream_ids"] = torch.full((Bk,), -1, dtype=torch.int64, device=dev)
            done = nets._done_bytes(static["done"], 1, Bk)
        elif model.training:
            static["stream_ids"] = torch.arange(Bk, dtype=torch.int64, device=dev)
        state = tuple(model.initial_state(Bk))
        seed_step = torch.zeros(2, dtype=torch.int64, device=dev)

        def step():
            if history is not None:
                history.fill(static["frame"], done, static["stream_ids"])
            return model(static, state)  # a [4, Bk] frame is an unstacked rollout: no second fill

        saved = model.action_sampler
        model.action_sampler = _DeviceStepSampler(seed_step)
        try:
            # warm up on a side stream (workspace, LSTM side stream, module loads), then capture
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(self.WARMUP_CALLS):
                    step()
            torch.cuda.current_stream(dev).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            # thread-local: another thread (a learner) may allocate or synchronise while this one captures
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                outputs, new_state = step()
        finally:
            model.action_sampler = saved
        self.captures += 1
        g = _Graph(graph, static, state, seed_step, getattr(model, "_ws", None), outputs, tuple(new_state))
        if history is not None:
            # The history the captured fill reads and writes: held, so its address (part of the key) stays this
            # buffer's for as long as the graph exists.
            g.history = history.buffer
            # The stacked scratch of the backends that restack (AtariNet fp32, ResNet fp32 / bf16), which the model
            # replaces for another shape.  nets._scratch sets this key only for those backends, so a fused backend
            # keeps no leftover scratch of an earlier shape alive here.
            g.scratch = model._scratch_buf if model._scratch_key == (1, Bk, dev, model.precision) else None
            g.real_rows = 0
        return g
