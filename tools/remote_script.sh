#!/bin/bash
# Run on the parameter-server node: install the cluster key, make every node reachable by its alias (node0 = PS, node1..), and
# replicate the repository (sources only; each node builds its own sm_90a extensions) to all workers.
# Idempotent: the ssh settings live in their own file (used with `ssh -F`), /etc/hosts entries are replaced, never duplicated.
# (role of the reference's tools/remote_script.sh:1-18)
set -euo pipefail
KEY=${1:?usage: remote_script.sh <ssh-key.pem> [user] [repo-dir]}
USER_=${2:-ubuntu}
REPO=${3:-draco_b200}
SSH_CFG=$HOME/.ssh/config.draco_cluster
mkdir -p ~/.ssh && cp "$KEY" ~/.ssh/id_cluster && chmod 600 ~/.ssh/id_cluster
cp "$(dirname "$0")/ssh_config.cluster" "$SSH_CFG" && chmod 600 "$SSH_CFG"
# ~/hosts lines are "<address>\t<alias>" with aliases node0, node1, ...: drop stale alias lines, then append the current ones
if [ -f ~/hosts ]; then
  sudo sh -c "grep -vE '[[:space:]]node[0-9]+\$' /etc/hosts > /tmp/hosts.new; cat /tmp/hosts.new $HOME/hosts > /etc/hosts"
fi
SSH="ssh -F $SSH_CFG"
tail -n +2 ~/hosts_alias | while read -r node; do
  [ -z "$node" ] && continue
  rsync -az -e "$SSH" --exclude .git --exclude gpurun_out --exclude '*.so' ~/"$REPO"/ "$USER_@$node:~/$REPO/" &
done
wait
# build the native code everywhere (PS included)
while read -r node; do
  [ -z "$node" ] && continue
  $SSH "$USER_@$node" "cd ~/$REPO && python -m draco_b200.build" < /dev/null &
done < ~/hosts_alias
wait
echo "cluster ready: $(wc -l < ~/hosts_alias) nodes"
