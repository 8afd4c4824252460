from offpolicy._b200.refpath import extend as _extend

_extend(__path__, 'algorithms', 'matd3', 'algorithm')
