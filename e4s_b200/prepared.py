"""Kernel-ready weights: the one cache every network keeps of its frozen parameters in kernel operand form (bf16 hi / lo
planes, folded BatchNorm, stacked MLPs, ...).

An entry is rebuilt when the device or any source tensor's (data_ptr, autograd version) differs from when it was built, so
``load_state_dict``, ``.to()`` and ordinary in-place ops are picked up.  Writes through ``.data`` (``param.data.copy_()``,
EMA accumulation loops) bump no version: call ``invalidate`` (``e4s_b200.invalidate_prepared``) after them.
"""
_ATTR = "_e4s_prepared"                     # {slot: (key, value)} on every module that holds an entry


def version_key(tensors, device) -> tuple:
    """(device, (data_ptr, version) of each tensor); a None entry (an absent bias or blur kernel) stays None."""
    return (str(device),) + tuple([None if t is None else (t.data_ptr(), t._version) for t in tensors])


def cached(module, slot: str, tensors, device, build):
    """``build()``'s value, kept on `module` under `slot` and rebuilt only when ``version_key(tensors, device)`` changes or
    the entry was invalidated.  Storing rebinds the module's attribute to a new dict instead of writing into the old one:
    DataParallel replicas start with a shallow copy of the original's attributes and must not write into its cache."""
    key = version_key(tensors, device)
    entries = vars(module).get(_ATTR, {})
    hit = entries.get(slot)
    if hit is not None and hit[0] == key:
        return hit[1]
    value = build()
    setattr(module, _ATTR, {**entries, slot: (key, value)})
    return value


def invalidate(module) -> None:
    """Drop every entry held by `module` and its submodules."""
    for m in module.modules():
        vars(m).pop(_ATTR, None)
