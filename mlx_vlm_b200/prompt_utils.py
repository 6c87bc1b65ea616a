"""Chat-template helpers of the reference's public surface (mlx_vlm/prompt_utils.py:
`get_message_json` :555-591, `get_chat_template` :594-826, `apply_chat_template` :829-995) for the
model families on the CUDA generate path — qwen2_vl, llava, llava_next, idefics2 ("list with image"
messages, prompt_utils.py:37,45,77,78) and qwen2_5_vl / idefics3 / smolvlm ("list with image first", :46,38,76) — plus the reference's text-only fallback for unknown types.
Behaviour is pinned against the reference's own module, executed, in tests/golden
(`chat_template_cases`).  Video / audio message kinds are outside the hot-path scope.
"""
from __future__ import annotations

import inspect
import json
from typing import Any, Dict, List, Optional, Tuple, Union

# model_type -> image entries come before the text entry?
_LIST_WITH_IMAGE: Dict[str, bool] = {"qwen2_vl": False, "qwen2_5_vl": True, "llava": False, "llava_next": False, "idefics2": False,
                                     "idefics3": True, "smolvlm": True}
_SINGLE_IMAGE_ONLY = {"llava_next"}     # prompt_utils.py:119-127
_IMAGE_KINDS = ("image", "image_url", "input_image")


def _text_of(content: Any) -> str:
    """Only the text parts of an OpenAI-style multimodal content list (prompt_utils.py:131-167)."""
    if isinstance(content, str):
        return content
    if isinstance(content, list):
        texts = []
        for part in content:
            if isinstance(part, dict) and part.get("type", "") in ("text", "input_text"):
                t = part.get("text", "") or part.get("content", "")
                if t:
                    texts.append(t)
        return " ".join(texts).strip()
    return str(content) if content else ""


def _role_content(item: Any) -> Optional[Tuple[str, Any]]:
    if isinstance(item, dict):
        return item.get("role", "user"), item.get("content")
    if hasattr(item, "role") and hasattr(item, "content"):
        return getattr(item, "role", "user"), getattr(item, "content", "")
    return None


def _tool_message(message: Dict[str, Any]) -> Dict[str, Any]:
    """Tool-calling messages pass through; JSON-string arguments become dicts (:189-218)."""
    out = dict(message)
    calls = out.get("tool_calls")
    if out.get("role") == "assistant" and calls and out.get("content") is None:
        out["content"] = ""
    if calls is None:
        return out
    fixed = []
    for call in calls:
        call = dict(call) if isinstance(call, dict) else call
        if isinstance(call, dict) and "function" in call:
            fn = dict(call["function"])
            args = fn.get("arguments", {})
            if isinstance(args, str):
                try:
                    fn["arguments"] = json.loads(args)
                except (json.JSONDecodeError, TypeError):
                    fn["arguments"] = {}
            call["function"] = fn
        fixed.append(call)
    out["tool_calls"] = fixed
    return out


def get_message_json(model_name: str, prompt: str, role: str = "user", skip_image_token: bool = False,
                     skip_audio_token: bool = False, num_images: int = 0, num_audios: int = 0,
                     **kwargs) -> Union[str, Dict[str, Any]]:
    name = model_name.lower()
    if name not in _LIST_WITH_IMAGE:
        raise ValueError(f"Unsupported model: {model_name}")
    if num_images > 1 and name in _SINGLE_IMAGE_ONLY:
        raise ValueError(f"Model {name} does not support multi-image chat. Please only use 1 image.")
    if kwargs.get("video"):
        raise NotImplementedError("video messages are outside this engine's hot-path scope")
    entries: List[Dict[str, Any]] = [{"type": "text", "text": prompt, "content": prompt}]
    if role == "user" and not skip_image_token and num_images > 0:
        images = [{"type": "image"}] * num_images
        entries = images + entries if _LIST_WITH_IMAGE[name] else entries + images
    if role == "user" and not skip_audio_token and num_audios > 0:
        entries = entries + [{"type": "audio"}] * num_audios
    return {"role": role, "content": entries}


def _marker(processor, attr: str, default: str) -> str:
    for holder in (processor, getattr(processor, "tokenizer", None)):
        tok = getattr(holder, attr, None) if holder is not None else None
        if isinstance(tok, str) and tok:
            return tok
    return default


def _plain_prompt(processor, messages, add_generation_prompt: bool, audio_token: str) -> str:
    """No chat template anywhere: "Role: text" lines (:690-737)."""
    image_token = _marker(processor, "image_token", "<image>")
    video_token = _marker(processor, "video_token", "<video>")
    markers = {image_token, video_token, audio_token, "<audio>", "<video>"}

    def flatten(content) -> str:
        if isinstance(content, str):
            return content
        if isinstance(content, dict):
            t = content.get("text", "") or content.get("content", "")
            return str(t) if t else ""
        if not isinstance(content, list):
            return str(content) if content is not None else ""
        parts: List[str] = []
        for item in content:
            if isinstance(item, dict):
                kind = item.get("type", "")
                if kind in _IMAGE_KINDS:
                    parts.append(image_token)
                elif kind in ("audio", "input_audio"):
                    parts.append("<audio>")
                elif kind in ("video", "input_video", "video_url"):
                    parts.append(video_token)
                else:
                    t = item.get("text", "") or item.get("content", "")
                    if t:
                        parts.append(str(t))
            elif item is not None:
                parts.append(str(item))
        out, after_marker = [], False
        for part in parts:
            if not part:
                continue
            is_marker = part in markers
            if after_marker and not is_marker and not part[0].isspace():
                out.append(" ")
            out.append(part)
            after_marker = is_marker
        return "".join(out).strip()

    rows = []
    for m in messages:
        if isinstance(m, dict):
            rows.append((m.get("role", "user"), flatten(m.get("content", ""))))
        else:
            rows.append(("user", m if isinstance(m, str) else str(m)))
    if not rows:
        return ""
    if len(rows) == 1 and rows[0][0] == "user":
        return rows[0][1]
    lines = []
    for role, text in rows:
        if role in ("system", "user", "assistant", "tool"):
            lines.append(f"{role.capitalize()}: {text}" if text else f"{role.capitalize()}:")
        else:
            lines.append(text or "")
    if add_generation_prompt:
        lines.append("Assistant:")
    return "\n".join(lines).strip()


def get_chat_template(processor, messages: List[Dict[str, Any]], add_generation_prompt: bool,
                      tokenize: bool = False, **kwargs) -> Any:
    """The processor's (or its tokenizer's) Jinja chat template when one exists, else the plain
    "Role: text" prompt (:594-826)."""
    override = kwargs.get("chat_template", None)
    audio_token = kwargs.get("audio_token", "<audio>")

    def has_template(obj) -> bool:
        return (obj is not None and hasattr(obj, "apply_chat_template")
                and (override is not None or getattr(obj, "chat_template", None) is not None))

    def plain():
        return _plain_prompt(processor, messages, add_generation_prompt, audio_token)

    try:
        target = None
        if has_template(processor):
            target = processor
        elif processor is not None and has_template(getattr(processor, "tokenizer", None)):
            target = processor.tokenizer
        if target is None:
            return plain()
        tkw = dict(kwargs)
        if "enable_thinking" not in tkw:
            try:
                params = inspect.signature(target.apply_chat_template).parameters
                if "enable_thinking" in params or any(p.kind == inspect.Parameter.VAR_KEYWORD
                                                      for p in params.values()):
                    tkw["enable_thinking"] = False
            except (TypeError, ValueError):
                pass
        if "thinking_mode" not in tkw and tkw.get("enable_thinking") is True:
            templates = [override, getattr(target, "chat_template", None),
                         getattr(getattr(target, "tokenizer", None), "chat_template", None)]
            for t in templates:
                vals = t.values() if isinstance(t, dict) else [t]
                if any(isinstance(v, str) and "thinking_mode" in v for v in vals):
                    tkw["thinking_mode"] = "enabled"
                    break
        try:
            return target.apply_chat_template(messages, tokenize=tokenize,
                                              add_generation_prompt=add_generation_prompt, **tkw)
        except ValueError as e:
            msg = str(e)
            if override is None and ("chat_template is not set" in msg
                                     or "no template argument was passed" in msg):
                return plain()
            raise
    except AttributeError:
        return plain()


def apply_chat_template(processor, config: Union[Dict[str, Any], Any],
                        prompt: Union[str, Dict[str, Any], List[Any]],
                        add_generation_prompt: bool = True, return_messages: bool = False,
                        num_images: int = 0, num_audios: int = 0, **kwargs):
    """prompt_utils.py:829-995: build per-model message dicts (image markers are attached to the
    user message that carries them, left-over images to the LAST user message), then render."""
    config = config if isinstance(config, dict) else config.__dict__
    model_type = config["model_type"]
    known = model_type.lower() in _LIST_WITH_IMAGE
    messages: List[Any] = []

    if not known:   # text-only formatting
        if isinstance(prompt, str):
            messages = [{"role": "user", "content": prompt}]
        elif isinstance(prompt, dict):
            m = dict(prompt)
            m["content"] = _text_of(m.get("content", ""))
            messages = [m]
        elif isinstance(prompt, list):
            for item in prompt:
                if isinstance(item, str):
                    messages.append({"role": "user", "content": item})
                    continue
                rc = _role_content(item)
                if rc is not None:
                    m = dict(item) if isinstance(item, dict) else {"role": rc[0]}
                    if rc[0] != "tool":
                        m["content"] = _text_of(rc[1])
                    messages.append(m)
        else:
            messages = [{"role": "user", "content": str(prompt)}]
        if return_messages:
            return messages
        return get_chat_template(processor, messages, add_generation_prompt, **kwargs)

    def is_tool(p, role) -> bool:
        return isinstance(p, dict) and ("tool_calls" in p or "tool_call_id" in p or role == "tool")

    if isinstance(prompt, str):
        messages.append(get_message_json(model_type, prompt, num_images=num_images,
                                         num_audios=num_audios, **kwargs))
    elif isinstance(prompt, dict):
        role = prompt.get("role", "user")
        if is_tool(prompt, role):
            messages.append(_tool_message(prompt))
        else:
            messages.append(get_message_json(model_type, _text_of(prompt["content"]), role,
                                             num_images=num_images, num_audios=num_audios, **kwargs))
    elif isinstance(prompt, list):
        last_user, explicit = -1, [0] * len(prompt)
        for i, p in enumerate(prompt):
            if isinstance(p, str):
                last_user = i
                continue
            rc = _role_content(p)
            if rc is not None and rc[0] not in ("system", "assistant", "tool"):
                last_user = i
                if isinstance(rc[1], list):
                    explicit[i] = sum(1 for it in rc[1]
                                      if isinstance(it, dict) and it.get("type") in _IMAGE_KINDS)
        left, n_img = num_images, []
        for c in explicit:
            c = min(c, left)
            n_img.append(c)
            left -= c
        if left and last_user >= 0:
            n_img[last_user] += left
        n_aud = [0] * len(prompt)
        if last_user >= 0:
            n_aud[last_user] = num_audios
        for i, p in enumerate(prompt):
            if isinstance(p, str):
                messages.append(get_message_json(model_type, p, skip_image_token=n_img[i] == 0,
                                                 skip_audio_token=n_aud[i] == 0, num_images=n_img[i],
                                                 num_audios=n_aud[i], **kwargs))
                continue
            rc = _role_content(p)
            if rc is None:
                continue
            role, content = rc
            if is_tool(p, role):
                messages.append(_tool_message(p))
            else:
                quiet = role in ("system", "assistant")
                messages.append(get_message_json(
                    model_type, _text_of(content), role, skip_image_token=n_img[i] == 0 or quiet,
                    skip_audio_token=n_aud[i] == 0 or quiet, num_images=n_img[i], num_audios=n_aud[i],
                    **kwargs))
    if return_messages:
        return messages
    return get_chat_template(processor, messages, add_generation_prompt, **kwargs)
