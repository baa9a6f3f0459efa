"""Caller side of the hot path (SURVEY.md 8f rank 2): the reference's local inference loop on top of the H100 model.

Mirrors ``ultravox/inference/base.py`` (``VoiceOutput``, ``InferenceChunk``, ``InferenceStats``, ``VoiceInference``) and
``ultravox/inference/infer.py:20-342`` (``LocalInference``: single / batch / streaming generation, conversation mode with
KV-cache reuse), same constructor arguments, method names and result types.  What differs, and why:

* decoding follows ref infer.py:319-328: greedy for ``temperature`` None / 0, multinomial sampling at a positive
  temperature (``do_sample=True``; top-k 50 like HF's ``GenerationConfig`` default), through the graph-captured decode engine;
* resampling to 16 kHz uses ``scipy.signal.resample_poly`` (``librosa`` - soxr_hq - is not in this image; the reference
  only pins the resulting frame / token counts, ref infer_test.py:112-132);
* ``infer_stream`` pushes tokens through a queue as the decode loop produces them (one ``InferenceChunk`` per decoded
  text delta); the conversation cache it keeps is the cache the generation returned.
"""
from __future__ import annotations

import abc
import copy
import dataclasses
import queue
import re
import threading
from typing import Dict, Generator, List, Optional, Tuple

import numpy as np
import torch

from .data_proc import VoiceSample
from .processing import DataCollatorForSeq2SeqWithAudio

SAMPLE_RATE = 16000
MAX_NEW_TOKENS = 1024
AUDIO_PLACEHOLDER = "<|audio|>"


@dataclasses.dataclass
class VoiceOutput:
    text: str
    input_tokens: int
    output_tokens: int
    thinking_content: Optional[str] = None


class InferenceMessage:
    pass


@dataclasses.dataclass
class InferenceChunk(InferenceMessage):
    text: str


@dataclasses.dataclass
class InferenceStats(InferenceMessage):
    input_tokens: int
    output_tokens: int


InferenceGenerator = Generator[InferenceMessage, None, None]


class VoiceInference(abc.ABC):
    @abc.abstractmethod
    def infer(self, sample: VoiceSample, max_tokens: Optional[int] = None, temperature: Optional[float] = None) -> VoiceOutput:
        ...

    def infer_batch(self, samples: List[VoiceSample], max_tokens: Optional[int] = None,
                    temperature: Optional[float] = None) -> List[VoiceOutput]:
        return [self.infer(s, max_tokens, temperature) for s in samples]

    def infer_stream(self, sample: VoiceSample, max_tokens: Optional[int] = None,
                     temperature: Optional[float] = None) -> InferenceGenerator:
        out = self.infer(sample, max_tokens, temperature)
        yield InferenceChunk(out.text)
        yield InferenceStats(out.input_tokens, out.output_tokens)


def resample_to_16k(audio: np.ndarray, sample_rate: int) -> np.ndarray:
    """Polyphase resampling of mono float PCM to 16 kHz (length = ceil(n * 16000 / sample_rate), like librosa's)."""
    if sample_rate == SAMPLE_RATE:
        return audio
    from math import gcd
    from scipy.signal import resample_poly
    g = gcd(SAMPLE_RATE, int(sample_rate))
    return resample_poly(audio.astype(np.float32), SAMPLE_RATE // g, int(sample_rate) // g).astype(np.float32)


class _TokenQueue:
    """Streamer protocol of ``UltravoxModel.generate`` (``put`` per step, ``end`` once): hands new tokens to another thread."""
    _END = object()

    def __init__(self):
        self.q: "queue.Queue" = queue.Queue()
        self.prompt_seen = False

    def put(self, tokens: torch.Tensor) -> None:
        if not self.prompt_seen:            # first call carries the prompt ids (as transformers' streamers get them)
            self.prompt_seen = True
            return
        self.q.put(int(tokens.reshape(-1)[0]))

    def end(self) -> None:
        self.q.put(self._END)

    def __iter__(self):
        while True:
            item = self.q.get()
            if item is self._END:
                return
            yield item


class LocalInference(VoiceInference):
    def __init__(self, model, processor, tokenizer, dtype: torch.dtype = torch.bfloat16, conversation_mode: bool = False,
                 chat_template: Optional[str] = None, enable_thinking: bool = False, thinking_regex: Optional[str] = None):
        if dtype != torch.bfloat16:
            raise ValueError("the H100 path computes in bf16")
        self.model = model.eval()
        self.tokenizer = tokenizer
        self.processor = processor
        self.dtype = dtype
        self.conversation_mode = conversation_mode
        self.past_messages: List[Dict[str, str]] = []
        self.past_key_values = None
        self.data_collator = DataCollatorForSeq2SeqWithAudio(tokenizer=tokenizer, include_alt_fields=False)
        self.chat_template = chat_template
        self.enable_thinking = enable_thinking
        self.thinking_regex = thinking_regex
        assert self.tokenizer.padding_side == "left"

    # -- conversation state -----------------------------------------------------------------------------------------
    def update_conversation(self, past_messages: Optional[List[Dict[str, str]]] = None, past_key_values=None) -> None:
        self.past_messages = list(past_messages or [])
        self.past_key_values = past_key_values

    def _get_sample_with_past(self, sample: Optional[VoiceSample]) -> VoiceSample:
        if sample is None:
            if not self.past_messages:
                raise ValueError("No past messages available to generate a response.")
            return VoiceSample(self.past_messages)
        sample = copy.copy(sample)
        sample.add_past_messages(self.past_messages)
        return sample

    def _build_past_messages(self, query_messages: List[Dict[str, str]], audio_token_len: int,
                             response_content: str) -> List[Dict[str, str]]:
        """The turn as later prompts must spell it: the audio placeholder becomes as many filler tokens as the clip
        occupied, so token positions keep matching the cached keys (ref infer.py:75-92)."""
        messages = [dict(m) for m in query_messages]
        if audio_token_len > 0:
            content = messages[-1]["content"]
            n = content.count(AUDIO_PLACEHOLDER)
            if n != 1:
                raise ValueError(f"Expected 1 audio placeholder, found {n}")
            messages[-1]["content"] = content.replace(AUDIO_PLACEHOLDER, self.tokenizer.eos_token * audio_token_len)
        messages.append({"role": "assistant", "content": response_content})
        return messages

    def _postprocess_response(self, text: str) -> Tuple[str, Optional[str]]:
        if not self.enable_thinking:
            return text, None
        if not self.thinking_regex:
            raise ValueError("thinking_regex is not set while enable_thinking is True")
        m = re.search(self.thinking_regex, text, re.DOTALL)
        if not m:
            raise ValueError(f"{self.thinking_regex} not matched in the response while thinking is enabled: {text}")
        return re.sub(self.thinking_regex, "", text, flags=re.DOTALL).strip(), m.group(1).strip()

    # -- feature preparation / generation ---------------------------------------------------------------------------
    def _dataproc(self, sample: VoiceSample, add_generation_prompt: bool = True) -> Dict[str, torch.Tensor]:
        text = self.tokenizer.apply_chat_template(sample.messages, add_generation_prompt=add_generation_prompt, tokenize=False,
                                                  chat_template=self.chat_template, enable_thinking=self.enable_thinking)
        audio = None
        if sample.audio is not None:
            a = sample.audio
            if a.dtype == np.int16:
                a = a / np.float32(32768.0)
            if a.dtype not in (np.float64, np.float32):
                raise ValueError("Audio must be float64 or float32 or int16")
            a = resample_to_16k(np.asarray(a), sample.sample_rate)
            audio = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
            if audio.ndim == 2:
                audio = audio.squeeze(0)
        inputs = self.processor(audio=audio, text=text, return_tensors="pt", sampling_rate=SAMPLE_RATE)
        dev = self.model.device
        return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in inputs.items()}

    def _terminators(self) -> List[int]:
        terminators = [self.tokenizer.eos_token_id]
        extra = getattr(self.tokenizer, "added_tokens_encoder", {})
        if "<|eot_id|>" in extra:
            terminators.append(self.tokenizer.convert_tokens_to_ids("<|eot_id|>"))
        return terminators

    @torch.inference_mode()
    def _generate(self, inputs: Dict[str, torch.Tensor], max_new_tokens: Optional[int] = None,
                  temperature: Optional[float] = None, streamer=None, past_key_values=None,
                  return_dict_in_generate: bool = True):
        # ref infer.py:319-328: temperature None -> model default (greedy here), 0 -> greedy, > 0 -> sample
        do_sample = temperature is not None and temperature > 0
        terminators = self._terminators()
        return self.model.generate(**inputs, max_new_tokens=max_new_tokens or MAX_NEW_TOKENS, eos_token_id=terminators,
                                   streamer=streamer, past_key_values=past_key_values, do_sample=do_sample,
                                   temperature=temperature if do_sample else None,
                                   return_dict_in_generate=return_dict_in_generate)

    # -- the three entry points ---------------------------------------------------------------------------------------
    def infer(self, sample: Optional[VoiceSample] = None, max_tokens: Optional[int] = None,
              temperature: Optional[float] = None) -> VoiceOutput:
        extended = self._get_sample_with_past(sample)
        inputs = self._dataproc(extended)
        input_len = int(inputs["input_ids"].shape[1])
        out = self._generate(inputs, max_tokens, temperature, past_key_values=self.past_key_values)
        new_tokens = out.sequences[0][input_len:]
        text, thinking = self._postprocess_response(self.tokenizer.decode(new_tokens, skip_special_tokens=True))
        if self.conversation_mode:
            tok_len = inputs.get("audio_token_len")
            n_audio = int(tok_len[0]) if tok_len is not None and len(tok_len) > 0 else 0
            self.update_conversation(self._build_past_messages(extended.messages, n_audio, text), out.past_key_values)
        return VoiceOutput(text, input_len, len(new_tokens), thinking_content=thinking)

    def infer_batch(self, samples: List[VoiceSample], max_tokens: Optional[int] = None,
                    temperature: Optional[float] = None) -> List[VoiceOutput]:
        """Left-padded batch through one generate call (no conversation mode, like the reference)."""
        assert not self.conversation_mode
        feats = []
        for s in samples:
            f = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in self._dataproc(s).items()}
            for key in list(f):
                if not key.startswith("audio") and torch.is_tensor(f[key]):
                    f[key] = f[key].squeeze(0)
            feats.append(f)
        batch = self.data_collator(feats)
        dev = self.model.device
        batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items() if v is not None}
        batch.pop("labels", None)
        input_len = int(batch["input_ids"].shape[1])
        seqs = self._generate(batch, max_tokens, temperature, return_dict_in_generate=False)
        outs = []
        for row in seqs:
            new_tokens = row[input_len:]
            text, thinking = self._postprocess_response(self.tokenizer.decode(new_tokens, skip_special_tokens=True))
            outs.append(VoiceOutput(text, input_len, len(new_tokens), thinking_content=thinking))
        return outs

    @torch.inference_mode()
    def infer_many(self, samples: List[VoiceSample], max_tokens: Optional[int] = None, temperature: Optional[float] = None,
                   slots: int = 8, max_len: Optional[int] = None) -> List[VoiceOutput]:
        """Serves independent samples through ``slots`` continuous-batching slots (``serving.SlotScheduler``): a finished reply
        frees its slot for the next sample at once, instead of a static batch decoding until its longest reply ends.  Same
        data processing, terminators and sampling rule as ``infer``; each result is what ``infer`` gives for that sample alone
        (no conversation mode, like ``infer_batch``).  Results come back in input order.  ``max_len`` is the slot capacity in
        positions (default: the longest prompt plus ``max_tokens``); a sample that does not fit raises ``ValueError``."""
        assert not self.conversation_mode
        from .serving import SlotScheduler
        feats = [self._dataproc(s) for s in samples]
        if not feats:
            return []
        max_new = max_tokens or MAX_NEW_TOKENS
        need = max(int(f["input_ids"].shape[1]) for f in feats) + max_new
        if max_len is not None and need > max_len:
            raise ValueError(f"a sample needs {need} positions (prompt + max_tokens); the slots hold {max_len}")
        sched = SlotScheduler(self.model, slots=slots, max_len=max_len or need, eos_token_ids=self._terminators())
        do_sample = temperature is not None and temperature > 0
        ids = [sched.submit(f, max_new_tokens=max_new, do_sample=do_sample, temperature=temperature if do_sample else None)
               for f in feats]
        res = sched.run()
        outs = []
        for f, rid in zip(feats, ids):
            input_len = int(f["input_ids"].shape[1])
            new_tokens = res[rid][0, input_len:]
            text, thinking = self._postprocess_response(self.tokenizer.decode(new_tokens, skip_special_tokens=True))
            outs.append(VoiceOutput(text, input_len, len(new_tokens), thinking_content=thinking))
        return outs

    def infer_stream(self, sample: Optional[VoiceSample] = None, max_tokens: Optional[int] = None,
                     temperature: Optional[float] = None) -> InferenceGenerator:
        extended = self._get_sample_with_past(sample)
        inputs = self._dataproc(extended)
        input_len = int(inputs["input_ids"].shape[1])
        streamer = _TokenQueue()
        result: Dict[str, object] = {}

        def run():
            try:
                result["out"] = self._generate(inputs, max_tokens, temperature, streamer=streamer,
                                               past_key_values=self.past_key_values)
            except BaseException as e:      # surface errors in the consumer thread instead of hanging it
                result["err"] = e
                streamer.end()

        dev = self.model.device

        def thread_main():
            with torch.cuda.device(dev):
                run()

        th = threading.Thread(target=thread_main)
        th.start()
        toks: List[int] = []
        text_so_far = ""
        for t in streamer:
            toks.append(t)
            text = self.tokenizer.decode(torch.tensor(toks), skip_special_tokens=True)
            delta, text_so_far = text[len(text_so_far):], text
            if delta:
                yield InferenceChunk(delta)
        th.join()
        if "err" in result:
            raise result["err"]  # type: ignore[misc]
        response, _ = self._postprocess_response(text_so_far)
        if self.conversation_mode:
            tok_len = inputs.get("audio_token_len")
            n_audio = int(tok_len[0]) if tok_len is not None and len(tok_len) > 0 else 0
            self.update_conversation(self._build_past_messages(extended.messages, n_audio, response),
                                     result["out"].past_key_values)  # type: ignore[union-attr]
        yield InferenceStats(input_len, len(toks))
