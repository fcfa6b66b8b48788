"""Chunked prefill in the paged inference engine (CPU tier): the step plans of the scheduler, greedy outputs equal to
the unchunked engine and to full recomputation, abort and recycle mid-prefill, and the rejected configurations.  fp32
engines run the reference attention paths."""
import math

import pytest
import torch

from colossalai_b200.inference import InferenceConfig, InferenceEngine
from colossalai_b200.inference.config import GenerationConfig
from colossalai_b200.inference.core.llm_engine import LLMEngine, prefix_caching_unsupported
from colossalai_b200.inference.struct import RequestStatus
from colossalai_b200.models import build_model, get_config

BS = 8
MAX_BS = 8
KW = dict(max_batch_size=MAX_BS, max_input_len=64, max_output_len=6, block_size=BS, dtype="fp32", ignore_eos=True)
LENS = [37, 5, 60, 18, 29, 9, 44, 3, 23, 51]          # more prompts than max_batch_size: they arrive in waves


def _prompt(i, L):
    return [(7 * i + 3 * j) % 500 + 3 for j in range(L)]


PROMPTS = [_prompt(i, L) for i, L in enumerate(LENS)]


def _naive_greedy(model, prompt, n_new):
    ids = list(prompt)
    for _ in range(n_new):
        with torch.no_grad():
            logits = model(input_ids=torch.tensor([ids]))["logits"]
        ids.append(int(logits[-1, : model.cfg.vocab_size].argmax()))
    return ids


def _engine(model, budget, **kw):
    return InferenceEngine(model, None, InferenceConfig(max_num_batched_tokens=budget, **{**KW, **kw}))


def _gen(eng, prompts, n_new):
    _, ids = eng.generate(prompts_token_ids=prompts, return_token_ids=True,
                          generation_config=GenerationConfig(max_new_tokens=n_new))
    return ids


def _trace(eng):
    """Record every step's plan: the chunks (request id, first position, tokens, prompt length), the output length of
    every decoding sequence fed, and every sequence's output length once the step's tokens are handed out."""
    rh = eng.request_handler
    steps = []
    schedule, update = rh.schedule, rh.update

    def traced_schedule():
        batch = schedule()
        chunked = batch is rh.prefill_bb
        seqs = rh.prefill_bb.seqs_li[: len(rh.prefill_chunks)] if chunked else []
        decoding = batch is rh.running_bb or rh.decode_in_step
        steps.append(dict(
            chunks=[(s.request_id, s.num_cached_tokens, n, s.input_len) for s, n in zip(seqs, rh.prefill_chunks)],
            decode={s.request_id: s.output_len for s in rh.running_bb.seqs_li} if decoding else {}))
        return batch

    def traced_update():
        steps[-1]["out"] = {s.request_id: s.output_len for s in rh.prefill_bb.seqs_li + rh.running_bb.seqs_li}
        return update()

    rh.schedule, rh.update = traced_schedule, traced_update
    return steps


@pytest.fixture(scope="module")
def llama():
    torch.manual_seed(0)
    return build_model("llama-tiny").float().eval()


@pytest.fixture(scope="module")
def reference(llama):
    """Greedy tokens of full recomputation and of the unchunked engine."""
    naive = [_naive_greedy(llama, p, 6) for p in PROMPTS]
    return naive, _gen(_engine(llama, None), PROMPTS, 6)


# ---------------------------------------------------------------------------------------------------- scheduler
@pytest.mark.parametrize("budget", [MAX_BS + BS, 4 * BS])
def test_step_plans(llama, reference, budget):
    eng = _engine(llama, budget)
    steps = _trace(eng)
    assert _gen(eng, PROMPTS, 6) == reference[1]
    started, finished, partial = [], [], None
    assert any(st["chunks"] and st["decode"] for st in steps), "no mixed step"
    for st in steps:
        chunks, decode, out = st["chunks"], st["decode"], st["out"]
        assert sum(n for _, _, n, _ in chunks) + len(decode) <= budget
        # every decoding sequence advances by one token in every step
        assert all(out[rid] == n + 1 for rid, n in decode.items())
        if partial is not None:                     # a partly prefilled prompt continues before any other
            assert chunks and chunks[0][0] == partial
        partial = None
        for j, (rid, start, n, L) in enumerate(chunks):
            assert start % BS == 0 and n > 0
            if start == 0:
                started.append(rid)
            if start + n < L:                       # a partial chunk: whole blocks, the step's last, samples nothing
                assert n % BS == 0 and j == len(chunks) - 1 and out[rid] == 0
                partial = rid
            else:
                assert out[rid] == 1
                finished.append(rid)
    assert sorted(finished) == list(range(len(PROMPTS)))
    assert finished == started                      # first come first served


def _steps_to_first_token(eng, prompt):
    eng.add_request(request_ids=[999], prompts_token_ids=[prompt])
    seq = eng.request_handler._find_sequence(999)
    n = 0
    while not seq.output_len:
        eng.step()
        n += 1
    return n


@pytest.mark.parametrize("budget", [MAX_BS + BS, 3 * BS])
@pytest.mark.parametrize("decoding", [0, 1, 3])
def test_long_prompt_takes_ceil_steps(llama, budget, decoding):
    """A prompt longer than the budget finishes in the predicted number of steps, the partial ones sampling nothing,
    while `decoding` streams take their token in every step."""
    eng = _engine(llama, budget, max_output_len=16)
    for i in range(decoding):
        eng.add_request(prompts_token_ids=[_prompt(100 + i, 3)])
    while any(lst for lst in eng.request_handler.waiting_list) or not eng.request_handler.prefill_bb.is_empty:
        eng.step()
    L = 60
    room = budget - decoding
    chunk = room // BS * BS
    expect = 1 + max(0, math.ceil((L - room) / chunk))
    assert expect > 1
    assert _steps_to_first_token(eng, _prompt(7, L)) == expect
    assert len(eng.request_handler.running_bb) == decoding + 1


# ---------------------------------------------------------------------------------------------------- outputs
@pytest.mark.parametrize("budget", [MAX_BS + BS, 3 * BS, 64])        # 64: at least the longest prompt
def test_greedy_equals_unchunked_and_recompute(llama, reference, budget):
    got = _gen(_engine(llama, budget), PROMPTS, 6)
    assert got == reference[1]
    assert got == reference[0]


def test_waves_arriving_mid_prefill(llama, reference):
    eng = _engine(llama, MAX_BS + BS)
    rh = eng.request_handler
    eng.add_request(request_ids=[0, 1], prompts_token_ids=PROMPTS[:2])
    eng.step()
    assert rh.prefill_bb.seqs_li and rh.prefill_bb.seqs_li[0].num_cached_tokens > 0       # mid-prefill
    eng.add_request(request_ids=list(range(2, 6)), prompts_token_ids=PROMPTS[2:6])
    eng.step()
    eng.add_request(request_ids=list(range(6, 10)), prompts_token_ids=PROMPTS[6:])
    done = []
    while rh.check_unfinished_reqs():
        done += eng.step()
    got = [s.input_token_id + s.output_token_id for s in sorted(done, key=lambda s: s.request_id)]
    assert got == reference[0]


SYS = [5, 9, 13, 200, 7, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33]     # > 2 blocks of 8


def test_prefix_caching_hits_plus_chunks(llama):
    waves = [[SYS + [40, 41] + _prompt(1, 20)], [SYS + _prompt(2 + i, 11 + 9 * i) for i in range(4)]]
    outs = []
    for budget in (None, MAX_BS + BS):
        eng = _engine(llama, budget, enable_prefix_caching=True)
        outs.append([_gen(eng, w, 6) for w in waves])
        assert eng.request_handler.cache_manager.prefix_cache_stats["hit_tokens"] > 0
    assert outs[0] == outs[1]
    for w, got in zip(waves, outs[1]):
        assert got == [_naive_greedy(llama, p, 6) for p in w]


def test_sliding_window_prompt_spanning_several_windows():
    torch.manual_seed(0)
    model = build_model(get_config("mistral-tiny", sliding_window=6)).float().eval()
    prompts = [_prompt(i, L) for i, L in enumerate([45, 13, 30])]
    got = _gen(_engine(model, MAX_BS + BS), prompts, 6)
    assert got == _gen(_engine(model, None), prompts, 6)
    assert got == [_naive_greedy(model, p, 6) for p in prompts]


def test_alibi():
    torch.manual_seed(0)
    model = build_model("baichuan-tiny").float().eval()
    model.fold_norm_head()
    prompts = [_prompt(i, L) for i, L in enumerate([41, 7, 26])]
    got = _gen(_engine(model, MAX_BS + BS), prompts, 5)
    assert got == _gen(_engine(model, None), prompts, 5)
    assert got == [_naive_greedy(model, p, 5) for p in prompts]


def test_speculative_decoding(llama):
    torch.manual_seed(1)
    drafter = build_model(get_config("llama-tiny", num_hidden_layers=1)).float().eval()
    prompts = [_prompt(i, L) for i, L in enumerate([40, 6, 27])]
    outs = []
    for budget in (None, MAX_BS + BS):
        eng = _engine(llama, budget, max_output_len=10, max_n_spec_tokens=4)
        eng.enable_spec_dec(drafter, n_spec_tokens=3)
        outs.append(_gen(eng, prompts, 10))
    for x, y in zip(*outs):
        assert x[:len(y)] == y[:len(x)]
    for p, g in zip(prompts, outs[1]):
        ref = _naive_greedy(llama, p, 10)
        assert g[:len(ref)] == ref


# ---------------------------------------------------------------------------------------------------- abort / recycle
def _mid_prefill(llama, **kw):
    eng = _engine(llama, MAX_BS + BS, enable_prefix_caching=True, **kw)
    rh = eng.request_handler
    total = rh.cache_manager.num_available_blocks
    eng.add_request(request_ids=[0], prompts_token_ids=[_prompt(3, 50)])
    eng.step()
    eng.step()
    seq = rh.prefill_bb.seqs_li[0]
    assert seq.num_cached_tokens == 2 * (MAX_BS + BS) and seq.output_len == 0
    return eng, seq, total


def test_abort_mid_prefill_frees_blocks_and_indexes_only_written_ones(llama):
    eng, seq, total = _mid_prefill(llama)
    mgr = eng.request_handler.cache_manager
    eng.request_handler.abort_sequence(0)
    assert seq.status == RequestStatus.ABORTED and eng.request_handler.prefill_bb.is_empty
    assert mgr.num_available_blocks == total
    assert len(mgr._block_entry) == 32 // BS                      # 4 written blocks of the 7 allocated
    assert len(mgr.match_prefix(_prompt(3, 50))) == 32 // BS
    assert not eng.request_handler.check_unfinished_reqs()


def test_recycle_mid_prefill_resets_the_count_and_finishes(llama):
    eng, seq, total = _mid_prefill(llama)
    rh = eng.request_handler
    rh._recycle_last()
    assert seq.status == RequestStatus.RECYCLED and seq.num_cached_tokens == 0 and rh.prefill_bb.is_empty
    assert rh.cache_manager.num_available_blocks == total
    assert len(rh.cache_manager._block_entry) == 32 // BS
    done = []
    while rh.check_unfinished_reqs():
        done += eng.step()
    assert [s.request_id for s in done] == [0]
    assert done[0].input_token_id + done[0].output_token_id == _naive_greedy(llama, _prompt(3, 50), 6)
    assert rh.cache_manager.prefix_cache_stats["hit_tokens"] == 32       # re-admitted onto its written blocks


@pytest.mark.parametrize("caching", [False, True])
def test_oversubscribed_cache_recycles_readmits_and_finishes(llama, caching):
    prompts = [_prompt(i, L) for i, L in enumerate([17, 30, 9])]
    kw = dict(max_batch_size=3, max_input_len=32, max_output_len=9, enable_prefix_caching=caching)
    eng = _engine(llama, 3 + BS + 5, **kw)
    mgr = eng.request_handler.cache_manager
    mgr._take_free_blocks(mgr.num_available_blocks - 9)        # fewer blocks than the sequences grow into
    recycled = []
    orig = eng.request_handler._recycle_last

    def spy():
        recycled.append(1)
        orig()

    eng.request_handler._recycle_last = spy
    got = _gen(eng, prompts, 9)
    assert recycled, "the cache was not over-subscribed"
    for p, g in zip(prompts, got):
        ref = _naive_greedy(llama, p, 9)           # a recycled sequence starts a new generation budget when re-admitted
        assert g[:len(ref)] == ref


# ---------------------------------------------------------------------------------------------------- rejections
@pytest.mark.parametrize("kw,msg", [
    (dict(max_num_batched_tokens=20), "multiple of block_size"),
    (dict(max_num_batched_tokens=0), "positive multiple"),
    (dict(max_num_batched_tokens=-16), "positive multiple"),
    (dict(max_num_batched_tokens=16, max_batch_size=9), "at least max_batch_size \\+ block_size"),
    (dict(max_num_batched_tokens=64, enable_streamingllm=True, generated_token_size=16), "enable_streamingllm"),
    (dict(max_num_batched_tokens=64, beam_width=2), "beam_width"),
])
def test_config_rejections(kw, msg):
    with pytest.raises(AssertionError, match=msg):
        InferenceConfig(block_size=8, **{"max_batch_size": 8, **kw})


def test_config_accepts_the_lower_bound():
    assert InferenceConfig(block_size=8, max_batch_size=8, max_num_batched_tokens=16).max_num_batched_tokens == 16


def test_rpc_engine_rejects_chunked_prefill():
    from colossalai_b200.inference.core.rpc_engine import RPCInferenceEngine

    cfg = InferenceConfig(max_batch_size=2, max_input_len=16, max_output_len=6, block_size=8, dtype="fp32",
                          max_num_batched_tokens=16)
    with pytest.raises(ValueError, match="RPC.*max_num_batched_tokens"):
        RPCInferenceEngine("llama-tiny", None, cfg)


@pytest.mark.parametrize("name,cfg_kw,model_kw", [
    ("fp8 cache", dict(dtype="bf16", kv_cache_dtype="fp8"), dict(head_dim=64)),
    ("fp32", dict(dtype="fp32"), dict(head_dim=64)),
    ("head_dim 16", dict(dtype="bf16"), dict()),
    ("MLA", dict(dtype="bf16"), None),
])
def test_cuda_engine_refuses_the_prefix_caching_envelope(name, cfg_kw, model_kw):
    """A CUDA engine refuses chunked prefill where it refuses prefix caching, with the same reason (the check runs
    at construction and needs no GPU)."""
    cfg = InferenceConfig(max_num_batched_tokens=64, **cfg_kw)
    model_cfg = get_config("deepseek_v3-tiny") if model_kw is None else get_config("llama-tiny", **model_kw)
    eng = LLMEngine.__new__(LLMEngine)
    eng.inference_config, eng.model, eng.model_config = cfg, torch.nn.Linear(1, 1), model_cfg
    eng.device = torch.device("cuda")
    reason = prefix_caching_unsupported(cfg, model_cfg)
    assert reason
    with pytest.raises(ValueError) as e:
        eng._verify_args()
    assert str(e.value) == f"max_num_batched_tokens: {reason}"
    eng.inference_config = InferenceConfig(max_num_batched_tokens=64, dtype="bf16")
    eng.model_config = get_config("llama-tiny", head_dim=128)
    eng._verify_args()                                                   # inside the envelope
