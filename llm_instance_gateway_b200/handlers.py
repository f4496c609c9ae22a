"""Host-side mirror of the ext-proc handler surface around the scheduler (pkg/ext-proc/handlers):
what Envoy sees does not change when the scheduler behind ``handlers.Scheduler`` is the GPU one.

    Server(pp, scheduler, targetPodHeader, datastore)          handlers/server.go:17-27
    Server.Process(request)                                    handlers/server.go:51-121
    Server.HandleRequestBody(reqCtx, body)                     handlers/request.go:19-121
    HandleRequestHeaders(reqCtx)                               handlers/request.go:123-143

Requests / responses are plain dicts shaped like the envoy ext_proc v3 messages (the protobuf
stack is not part of the hot path and is not rebuilt here):
    {"request_headers": {...}} | {"request_body": {"body": bytes}}
 -> {"request_headers": {"response": {"clear_route_cache": True}}}
  | {"request_body": {"response": {"header_mutation": {"set_headers": [...]}, "body_mutation": {"body": bytes}}}}
  | {"immediate_response": {"status": {"code": 429}}}
Used by tests/test_hermetic_replay.py, the replay of pkg/ext-proc/test/hermetic_test.go:27-139.
"""
from __future__ import annotations

import json
import math
from dataclasses import dataclass, field
from typing import Any, Dict, Optional

from .backend import DRAW_DOMAIN, IsCritical, Pod, RandomWeightedDraw, SplitMixSource
from .scheduling import LLMRequest, StatusError


@dataclass
class RequestContext:                        # handlers/server.go:123-127
    TargetPod: Pod = field(default_factory=Pod)
    Model: str = ""


class GoError(Exception):
    """A plain Go error (fmt.Errorf): status.Code() of it is Unknown."""
    code = "Unknown"


def _go_number(x: float) -> str:
    """encoding/json's float64 formatting (json.Unmarshal turns every JSON number into float64)."""
    if x != x or x in (math.inf, -math.inf):
        raise ValueError("json: unsupported value")
    if x == int(x) and abs(x) < 1e21:
        return str(int(x))
    r = repr(float(x))
    if "e" in r:
        mant, exp = r.split("e")
        ex = int(exp)
        if -7 < ex < 21:
            return format(x, "f").rstrip("0").rstrip(".")
        return f"{mant}e{'-' if ex < 0 else '+'}{abs(ex):02d}" if abs(ex) < 10 else f"{mant}e{'-' if ex < 0 else '+'}{abs(ex)}"
    return r


def go_json_marshal(v: Any) -> bytes:
    """json.Marshal of what json.Unmarshal(…, &map[string]interface{}) produced: map keys sorted,
    no whitespace, numbers as float64, HTML-escaping of <, >, &."""
    def enc(x):
        if x is None:
            return "null"
        if x is True:
            return "true"
        if x is False:
            return "false"
        if isinstance(x, (int, float)):
            return _go_number(float(x))
        if isinstance(x, str):
            s = json.dumps(x, ensure_ascii=False)
            return s.replace("<", "\\u003c").replace(">", "\\u003e").replace("&", "\\u0026")
        if isinstance(x, list):
            return "[" + ",".join(enc(e) for e in x) + "]"
        if isinstance(x, dict):
            return "{" + ",".join(f"{enc(k)}:{enc(x[k])}" for k in sorted(x)) + "}"
        raise TypeError(type(x))
    return enc(v).encode("utf-8")


def HandleRequestHeaders(reqCtx: RequestContext) -> Dict[str, Any]:          # handlers/request.go:123-143
    return {"request_headers": {"response": {"clear_route_cache": True}}}


class Server:
    def __init__(self, pp, scheduler, targetPodHeader: str, datastore, seed: int = 0):   # handlers/server.go:17-27
        self.scheduler = scheduler
        self.targetPodHeader = targetPodHeader
        self.pp = pp
        self.datastore = datastore
        self._seed = seed
        self._n = 0

    def HandleRequestBody(self, reqCtx: RequestContext, body: bytes) -> Dict[str, Any]:   # handlers/request.go:19-121
        try:
            rb = json.loads(body)                                            # request.go:24-28
        except Exception as ex:
            raise GoError(f"error unmarshaling request body: {ex}")
        if not isinstance(rb, dict):
            raise GoError("error unmarshaling request body: not an object")
        model = rb.get("model")
        if not isinstance(model, str):                                       # request.go:32-35
            raise GoError("model not found in request")
        modelName = model
        resolves = getattr(self.scheduler, "ResolvesModels", None)
        if callable(resolves) and resolves():
            # a scheduler holding the InferenceModels resolves on the device; its errors are already
            # the ones below (the Go adapter's patch 0004 takes the same branch)
            modelName, targetPod = self.scheduler.ScheduleModel(model)
            return self._respond(reqCtx, rb, body, LLMRequest(Model=model, ResolvedTargetModel=modelName), targetPod)
        modelObj = self.datastore.FetchModelData(model)                     # request.go:42-45
        if modelObj is None:
            raise GoError(f"error finding a model object in InferenceModel for input {model}")
        self._n += 1
        key = self._n
        if len(modelObj.Spec.TargetModels) > 0:                              # request.go:46-51
            modelName = RandomWeightedDraw(modelObj, SplitMixSource(self._seed ^ key ^ DRAW_DOMAIN))
            if modelName == "":
                raise GoError(f"error getting target model name for model {modelObj.Name}")
        llmReq = LLMRequest(Model=model, ResolvedTargetModel=modelName, Critical=IsCritical(modelObj))   # request.go:52-56
        try:
            targetPod = self.scheduler.Schedule(llmReq)                      # request.go:71-74
        except StatusError as err:
            raise StatusError(err.code, f"failed to find target pod: {err}")   # %w keeps the status code
        return self._respond(reqCtx, rb, body, llmReq, targetPod)

    def _respond(self, reqCtx: RequestContext, rb: Dict[str, Any], body: bytes, llmReq: LLMRequest,
                 targetPod) -> Dict[str, Any]:
        requestBody = body
        if llmReq.Model != llmReq.ResolvedTargetModel:                       # request.go:60-69
            rb["model"] = llmReq.ResolvedTargetModel
            requestBody = go_json_marshal(rb)
        reqCtx.Model = llmReq.Model
        reqCtx.TargetPod = targetPod
        headers = [                                                           # request.go:80-96
            {"header": {"key": self.targetPodHeader, "raw_value": targetPod.Address.encode()}},
            {"header": {"key": "Content-Length", "raw_value": str(len(requestBody)).encode()}},
        ]
        return {"request_body": {"response": {"header_mutation": {"set_headers": headers},
                                              "body_mutation": {"body": requestBody}}}}

    def Process(self, reqCtx: RequestContext, request: Dict[str, Any]) -> Dict[str, Any]:   # handlers/server.go:51-121
        """One iteration of the stream loop: returns the response to send, or raises the status
        error the stream is closed with."""
        try:
            if "request_headers" in request:
                return HandleRequestHeaders(reqCtx)
            if "request_body" in request:
                return self.HandleRequestBody(reqCtx, request["request_body"]["body"])
            raise StatusError("Unknown", "unknown request type")
        except (StatusError, GoError) as err:
            if getattr(err, "code", "Unknown") == "ResourceExhausted":      # server.go:97-109
                return {"immediate_response": {"status": {"code": 429}}}    # StatusCode_TooManyRequests
            raise StatusError(getattr(err, "code", "Unknown"), f"failed to handle request: {err}")   # server.go:110-112


def NewServer(pp, scheduler, targetPodHeader: str, datastore, **kw) -> Server:   # handlers/server.go:17
    return Server(pp, scheduler, targetPodHeader, datastore, **kw)
