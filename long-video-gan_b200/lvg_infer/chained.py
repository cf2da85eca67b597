"""Chained low-res -> super-res inference for long videos (SURVEY.md 8f N4; BASELINE.json configs[4]).

The reference's ``generate.py:56-88`` runs the low-res generator over the whole sequence, then walks
``sres_G.sample_video_segments`` ONE 16-frame segment at a time at batch 1 (``generator_sres.py:662-681``) and finally
``torch.cat``s every high-res segment on the device (4096 frames at 256x144 fp32 = 1.8 GB) before the encoder sees the first
frame. A single segment leaves most of the SMs idle (the 64-channel layers launch fewer CTAs than there are
SMs) and the device-side concatenation is what bounds the video length.

``generate_video`` keeps the reference's arithmetic -- same ``latent_z`` for every segment, same windows with
``temporal_context`` frames on either side -- and changes the schedule:

* ``segments_per_batch`` windows are stacked along the batch axis of ONE super-res forward (the network treats batch items
  independently in eval mode: per-sample modulated convolutions, no batch statistics), so the kernels of
  ``torch_utils.ops`` run at training-like sizes;
* finished segments are converted to ``uint8`` on the device (the ``[-1, 1] -> [0, 255]`` mapping of
  ``utils.write_video_grid``, utils.py:146-186 -- 4x fewer bytes over PCIe) and copied to pinned host memory on a side
  stream while the next batch computes; the consumer (an encoder, a file) receives frames in order through a callback or
  an iterator and nothing but two batches of segments is ever resident;
* the super-res forward of a full batch can be captured in a CUDA graph (``graph=True``; the last, shorter batch runs eagerly).

The generators are passed in (unpickled reference modules importing ``torch_utils.ops`` from this package, or any module
with the same call signature): ``lres_G(batch, seq_length, generator_emb=...)``, ``sres_G.SG3(latent_z, lr_segment)``,
``sres_G.sample_latent_z(batch, generator)``, ``sres_G.temporal_context``.
"""
import torch


def segment_windows(lr_video, segment_length, temporal_context):
    """The reference's windows: ``lr_video.unfold(2, segment_length + 2*context, segment_length)`` as a list of views
    ``[N, C, segment_length + 2*context, H, W]`` (generator_sres.py:675-679)."""
    n_out = lr_video.size(2) - 2 * temporal_context
    if n_out <= 0 or n_out % segment_length != 0:
        raise ValueError('low-res length must be segments * segment_length + 2 * temporal_context')
    size = segment_length + 2 * temporal_context
    return [lr_video[:, :, s:s + size] for s in range(0, n_out, segment_length)]


def to_uint8(video):
    """``[-1, 1]`` float video -> uint8 (the value mapping of ``utils.write_video_grid`` / ``save_image_grid``)."""
    return (video.float() * 127.5 + 128).clamp_(0, 255).to(torch.uint8)


class _HostRing:
    """Two pinned host buffers + a copy stream: segment batch k is copied out while batch k+1 computes."""

    def __init__(self, shape, dtype, device):
        self.cuda = device.type == 'cuda'
        self.bufs = [torch.empty(shape, dtype=dtype, pin_memory=self.cuda) for _ in range(2)]
        self.events = [None, None]
        self.stream = torch.cuda.Stream(device) if self.cuda else None
        self.k = 0

    def push(self, tensor):
        """Start the copy of `tensor` (device) into the next host buffer; returns (host view, wait())."""
        i = self.k % 2
        self.k += 1
        host = self.bufs[i][:tensor.shape[0]]
        if not self.cuda:
            host.copy_(tensor)
            return host, (lambda: None)
        self.stream.wait_stream(torch.cuda.current_stream(tensor.device))
        with torch.cuda.stream(self.stream):
            host.copy_(tensor, non_blocking=True)
            tensor.record_stream(self.stream)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return host, ev.synchronize


@torch.no_grad()
def generate_video(lres_G, sres_G, seq_length, generator=None, segment_length=16, segments_per_batch=8, as_uint8=True,
                   graph=False, sink=None):
    """Generates ``seq_length`` frames at super-res resolution for ONE video (``generate.py`` runs batch 1).

    Returns ``(lr_video, chunks)``: the low-res video (device tensor, ``temporal_context`` frames of lead-in and lead-out
    included, as in ``generate.py``) and an iterator of ``(first_frame_index, frames)`` with host tensors
    ``[3, frames, H, W]`` in temporal order (uint8 when ``as_uint8``, else the network's float output),
    ``segments_per_batch * segment_length`` frames at a time, the last chunk cut to ``seq_length``. A chunk's memory is
    reused two chunks later: consume (encode, write) it before asking for the one after next. With a ``sink`` the
    chunks are passed to ``sink(first_frame_index, frames)`` instead and the iterator comes back exhausted.
    """
    it = _generate(lres_G, sres_G, seq_length, generator, segment_length, segments_per_batch, as_uint8, graph)
    lr_video = next(it)
    if sink is not None:
        for first, frames in it:
            sink(first, frames)
    return lr_video, it


def _generate(lres_G, sres_G, seq_length, generator, segment_length, segments_per_batch, as_uint8, graph):
    ctx = int(sres_G.temporal_context)
    lr_len = -(-seq_length // segment_length) * segment_length + 2 * ctx                  # generate.py:60-61
    lr_video = lres_G(1, lr_len, generator_emb=generator)
    yield lr_video
    device = lr_video.device
    latent_z = sres_G.sample_latent_z(1, generator)                                        # ONE latent for the whole video
    windows = segment_windows(lr_video, segment_length, ctx)
    k = max(1, int(segments_per_batch))
    z_full = latent_z.expand(k, *latent_z.shape[1:]).contiguous()

    def run(z, lr_batch):
        hr = sres_G.SG3(z, lr_batch)                                                       # [k, 3, segment_length, H, W]
        hr = hr.permute(1, 0, 2, 3, 4).reshape(hr.shape[1], -1, hr.shape[3], hr.shape[4])  # segments are consecutive in time
        return to_uint8(hr) if as_uint8 else hr.float()

    graphed = None
    static_lr = None
    ring = None
    pending = None                                                                         # (first frame, host view, wait)
    for b0 in range(0, len(windows), k):
        chunk = windows[b0:b0 + k]
        lr_batch = torch.cat(chunk, dim=0)                                                 # windows overlap: a copy, k * (L + 2c) frames
        if graph and device.type == 'cuda' and len(chunk) == k:
            if graphed is None:
                from lvg_dist.flat_optim import GraphedCallable
                static_lr = lr_batch.clone()
                graphed = GraphedCallable(lambda lr: run(z_full, lr), static_lr)
            out = graphed(lr_batch).clone()             # the graph's output buffer is overwritten by the next replay
        else:
            out = run(z_full[:len(chunk)], lr_batch)
        if ring is None:
            ring = _HostRing((k * segment_length,) + tuple(out.permute(1, 0, 2, 3).shape[1:]), out.dtype, device)
        # frames-major on the host: [frames, 3, H, W] slices are contiguous for an encoder
        host, wait = ring.push(out.permute(1, 0, 2, 3).contiguous())
        if pending is not None:                                                            # hand out batch k-1 while batch k is in flight
            yield _finish(pending, seq_length)
        pending = (b0 * segment_length, host, wait)
    if pending is not None:
        yield _finish(pending, seq_length)


def _finish(pending, seq_length):
    first, host, wait = pending
    wait()
    frames = host[:max(0, min(host.shape[0], seq_length - first))]
    return first, frames.permute(1, 0, 2, 3)
